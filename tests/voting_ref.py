"""Plain NumPy/fp64 restatement of LightGBM 3.2's voting-parallel tree learner (VotingParallelTreeLearner, the PV-Tree algorithm) over R
row shards, built on split_scan_ref.py's scans.  It imports neither mmlspark_b200 nor oracle.

Per round, for each new leaf (smaller / larger by global counts):
1. every rank scans its local histogram of each of its flagged features with the local config (min_data_in_leaf // R,
   min_sum_hessian_in_leaf / R), the leaf's local sums and its true local row count; the scan sets that rank's is_splittable flags;
2. every rank sends its top_k candidates by (gain desc, real feature asc) as (feature, gain, left_count, right_count);
3. the vote, the same on every rank: mean = global count / R in fp32 (score_t); a record weighs gain * (left_count + right_count) / mean;
   each feature keeps its largest weight (strict >); the top_k features by (weight desc, feature asc) with a finite weight are voted;
4. the voted features alone are scanned on the global histogram with the training config, the leaf's global sums and its global count,
   whatever the local flags.  The best of those is the leaf's split, and the tree grows as in the data-parallel learner: the recorded
   counts are the split's hessian-rebuilt left count and the leaf's global count minus it.
One rank is the serial learner (true counts, no vote).  Local histograms are exact for every feature (upstream keeps a stale buffer for a
feature that is locally unsplittable in the parent; see DESIGN.md §5)."""
import math

import numpy as np

import split_scan_ref as ref

NEG_INF = ref.NEG_INF


def local_params(p, R):
    q = ref.Params(**{k: getattr(p, k) for k in ref.Params.DEFAULTS})
    q.min_data_in_leaf = p.min_data_in_leaf // R
    q.min_sum_hessian_in_leaf = p.min_sum_hessian_in_leaf / R
    return q


def local_top_k(scans, top_k):
    """records (feature, gain, left_count, right_count) of the top_k candidates of one rank's scans; -inf candidates send nothing"""
    cands = sorted((s for s in scans.values() if s.gain > NEG_INF), key=lambda s: (-s.gain, s.feature))[:top_k]
    return [(s.feature, s.gain, s.left_count, s.num_data - s.left_count) for s in cands]


def vote(records, global_count, R, top_k):
    """GlobalVoting over every rank's records, in rank order: the voted features, best first"""
    mean = float(np.float32(global_count) / np.float32(R))
    best = {}
    for f, gain, lc, rc in records:
        if f < 0:
            continue
        w = gain * (lc + rc) / mean
        if w > best.get(f, NEG_INF):
            best[f] = w
    top = sorted(best.items(), key=lambda kv: (-kv[1], kv[0]))[:top_k]
    return [f for f, w in top if w > NEG_INF]


def _scan_feature(bins, g, h, rows, f, sum_g, sum_h, num_data, p):
    col = bins[rows, f.real_index].astype(np.int64)
    hg = np.bincount(col, weights=g[rows], minlength=f.num_bin)
    hh = np.bincount(col, weights=h[rows], minlength=f.num_bin)
    if f.is_cat:
        s = ref.find_best_categorical(hg, hh, f.num_bin, sum_g, sum_h, num_data, p, f.real_index)
    else:
        s = ref.find_best_numerical(hg, hh, f.num_bin, f.missing_type, f.offset, sum_g, sum_h, num_data, p, f.real_index)
    s.num_data = num_data
    return s


def grow_voting_tree(bins, g, h, features, p, num_leaves, rank_of_row, R, top_k):
    """bins: [rows][real features]; g/h: fp64 values on an exact grid; rank_of_row: the rank holding each row.  Returns the tree arrays as
    split_scan_ref.grow_tree does, with `voted`: per round the (smaller, larger) voted feature lists (larger None at the root)."""
    if R == 1:
        T = ref.grow_tree(bins, g, h, features, p, num_leaves)
        T["voted"] = []
        return T
    assert top_k > 0
    top_k = min(top_k, len(features))
    n = len(g)
    by_real = {f.real_index: f for f in features}
    lp = local_params(p, R)
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags=[{f.real_index: True for f in features} for _ in range(R)])]
    T = dict(split_feature=[], threshold_bin=[], default_left=[], is_cat=[], cat_bins=[], split_gain=[], left_child=[], right_child=[],
             internal_value=[], internal_weight=[], internal_count=[], voted=[])
    parent_of = [-1]
    new_leaves = [0]
    while True:
        counts = [leaves[l]["count"] for l in new_leaves]
        go = len(leaves) < num_leaves and not all(c < p.min_data_in_leaf * 2 for c in counts)
        if go:
            if len(new_leaves) == 2:
                a, b = new_leaves
                order = [a, b] if leaves[a]["count"] < leaves[b]["count"] else [b, a]
            else:
                order = new_leaves
            voted_round = []
            for l in order:
                L = leaves[l]
                records = []
                for r in range(R):
                    rows = L["rows"][rank_of_row[L["rows"]] == r]
                    lg, lh = math.fsum(g[rows]), math.fsum(h[rows])
                    scans = {}
                    for f in features:
                        if L["flags"][r][f.real_index]:
                            scans[f.real_index] = _scan_feature(bins, g, h, rows, f, lg, lh, len(rows), lp)
                    for fi, s in scans.items():
                        L["flags"][r][fi] = s.splittable
                    records += local_top_k(scans, top_k)
                voted = vote(records, L["count"], R, top_k)
                voted_round.append(voted)
                scans = {fi: _scan_feature(bins, g, h, L["rows"], by_real[fi], L["sum_g"], L["sum_h"], L["count"], p) for fi in voted}
                L["best"] = ref.best_of_leaf(scans)
            T["voted"].append((voted_round[0], voted_round[1] if len(voted_round) > 1 else None))
        else:
            for l in new_leaves:
                leaves[l]["best"] = None
        if len(leaves) >= num_leaves:
            break
        pick = None
        for li, L in enumerate(leaves):
            b = L["best"]
            if b is None:
                continue
            if pick is None or ref.better_split(b.gain, b.feature, leaves[pick]["best"].gain, leaves[pick]["best"].feature):
                pick = li
        if pick is None or not leaves[pick]["best"].gain > 0.0:
            break
        L, s = leaves[pick], leaves[pick]["best"]
        f = by_real[s.feature]
        col = bins[L["rows"], f.real_index].astype(np.int64)
        left = ref.goes_left(col, f, s)
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
        T["internal_value"].append(L["value"]); T["internal_weight"].append(L["weight"])
        T["internal_count"].append(L["count"])
        lcount, rcount = s.left_count, L["count"] - s.left_count      # hessian-rebuilt global counts of the split
        flags = [dict(fl) for fl in L["flags"]]
        R_ = dict(rows=L["rows"][~left], sum_g=L["sum_g"] - s.left_g, sum_h=sum_h2 - s.left_h - ref.K_EPS, count=rcount, best=None,
                  value=0.0 if math.isnan(right_out) else right_out, weight=sum_h2 - s.left_h - ref.K_EPS, flags=[dict(fl) for fl in flags])
        L.update(rows=L["rows"][left], sum_g=s.left_g, sum_h=s.left_h - ref.K_EPS, count=lcount, best=None,
                 value=0.0 if math.isnan(left_out) else left_out, weight=s.left_h - ref.K_EPS, flags=flags)
        leaves.append(R_)
        parent_of[pick] = node
        parent_of.append(node)
        new_leaves = [pick, nl]
    T["num_leaves"] = len(leaves)
    T["leaf_value"] = [L["value"] if abs(L["value"]) > ref.K_ZERO else 0.0 for L in leaves]
    T["leaf_weight"] = [L["weight"] for L in leaves]
    T["leaf_count"] = [L["count"] for L in leaves]
    T["internal_value"] = [v if abs(v) > ref.K_ZERO else 0.0 for v in T["internal_value"]]
    return T
