"""One NumPy restatement of LightGBM 3.2's leaf-wise tree growth (SerialTreeLearner::Train, and VotingParallelTreeLearner's leaf search)
that every split option plugs into: the scans of split_scan_ref.py, the random thresholds of extra_trees_ref.py, the bounds and penalty of
monotone_ref.py, the set masks of interaction_ref.py, the node samples of bynode_ref.py and the vote of voting_ref.py.  Each of those
modules keeps its own rule; the rounds, the pick, the tree arrays and the children live here once.  It imports neither mmlspark_b200 nor
oracle.

Growth, with learning_rate 1 and no bias:
- A round scans the new leaves (the root, then the two children of the last split) unless the tree is full, every new leaf holds fewer
  than min_data_in_leaf * 2 rows, or (max_depth > 0) the new leaves are at max_depth, as the engine's round controller decides.  The
  smaller leaf (fewer rows; the right one on a tie) is scanned first: that is the order of the extra-trees and the by-node draws.
- A scan searches every feature whose is_splittable flag is set (the tree's feature_fraction sample at the root, then inherited), and
  sets the flag.  The leaf's best split is taken over the scanned features its interaction mask allows and its node sample holds.
- The leaf with the best split (SplitInfo::operator>, then the first leaf) splits if its gain is positive.  Its children take the split's
  sums, outputs (clamped to the leaf's monotone bounds), the narrowed bounds, the narrowed mask and the parent's flags.  Their counts are
  their rows, or under voting and data-parallel learning the split's hessian-rebuilt global counts."""
import math

import numpy as np

import extra_trees_ref as X3
import interaction_ref as I
import monotone_ref as M
import split_scan_ref as ref
import voting_ref as V

NO_BOUNDS = (-math.inf, math.inf)


def scan_leaf(bins, g, h, rows, sum_g, sum_h, num_data, features, flags, p, streams=None, mono=None, penalty=0.0, bounds=NO_BOUNDS,
              depth=0):
    """All (feature) searches of one leaf over its rows: {real_index: Scan} for the features whose flag is set.  With `streams` (an
    extra_trees_ref.Streams) every scanned feature draws once; with a `mono` list the scans are the constrained ones at the leaf's bounds,
    and a monotone feature's shifted gain is multiplied by the penalty factor at the leaf's depth.  The candidates keep their own gains:
    undecided compares those with min_gain_shift, which the scan does before the penalty; within a leaf every monotone feature has the
    same factor."""
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
            if mono is None:
                out[fi] = X3.find_best_categorical(hg, hh, f.num_bin, sum_g, sum_h, num_data, p, fi, t)
            else:
                out[fi] = M.find_best_categorical(hg, hh, f.num_bin, sum_g, sum_h, num_data, p, fi, bounds, t)
        else:
            t = None if streams is None else streams.draw(f, X3.numerical_range(f.num_bin))
            if mono is None:
                out[fi] = X3.find_best_numerical(hg, hh, f.num_bin, f.missing_type, f.offset, sum_g, sum_h, num_data, p, fi, t)
            else:
                s = out[fi] = M.find_best_numerical(hg, hh, f.num_bin, f.missing_type, f.offset, sum_g, sum_h, num_data, p, fi, bounds,
                                                    mono[fi], t)
                if mono[fi] != 0 and s.gain != ref.NEG_INF:
                    s.gain *= M.penalty_factor(depth, penalty)
    return out


def _vote(bins, g, h, L, features, p, voting):
    """VotingParallelTreeLearner's leaf search: every rank scans its rows with the local config and sets its own flags, the ranks vote on
    their top_k records, and the voted features alone are scanned over every row of the leaf.  Returns (voted, global scans)."""
    rank_of_row, R, top_k = voting
    lp = V.local_params(p, R)
    records = []
    for r in range(R):
        rows = L["rows"][rank_of_row[L["rows"]] == r]
        scans = scan_leaf(bins, g, h, rows, math.fsum(g[rows]), math.fsum(h[rows]), len(rows), features, L["flags"][r], lp)
        for fi, s in scans.items():
            L["flags"][r][fi] = s.splittable
            s.num_data = len(rows)
        records += V.local_top_k(scans, top_k)
    voted = V.vote(records, L["count"], R, top_k)
    flags = {f.real_index: f.real_index in voted for f in features}
    return voted, scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, flags, p)


def grow_tree(bins, g, h, features, p, num_leaves, *, used=None, streams=None, mono=None, penalty=0.0, constraints=None, sampler=None,
              max_depth=-1, voting=None, estimated_counts=False):
    """One tree.  bins: [rows][real features] bin indices; g/h: fp64 values on an exact grid.  The options, each off by default:
    - used: the real indices the tree's feature_fraction sample holds (None: every feature);
    - streams: an extra_trees_ref.Streams, which turns extra trees on and carries the feature streams from tree to tree;
    - mono: the monotone constraint list indexed by real feature (a non-empty list, all zeros included, runs the constrained scans), with
      `penalty` the monotone_penalty;
    - constraints: the interaction constraint sets (None: one set of every feature, which allows every feature at every leaf);
    - sampler: a bynode_ref.ColSampler, which takes the tree's feature_fraction sample (instead of `used`) and every leaf's node sample;
    - max_depth: > 0 stops the rounds whose leaves are at that depth;
    - voting: (rank_of_row, R, top_k), the rank holding each row; one rank is the serial learner;
    - estimated_counts: the children's counts are the split's hessian-rebuilt counts, as the data-parallel learner keeps them (voting
      always does).
    Returns the tree arrays as the model text prints them (bins instead of threshold values, bin sets instead of categories) and:
    rounds: per round, (leaf, leaf state, scans) in scan order; picks: per pick, every leaf's best split; scanned_counts: per round, the
    (leaf, row count) pairs in (left, right) order; leaf_rows: every leaf's rows (indices into g), ascending; bounds, masks, branches: every leaf's final monotone bounds, set mask and split
    features from the root; scan_masks and node_rounds: per round, each scanned leaf's mask and its (mask, node sample) in scan order;
    draws: the sampler's draws of the tree, its tree draw included; voted: per round, the (smaller, larger) voted feature lists (larger
    None at the root)."""
    features = sorted(features, key=lambda f: f.real_index)
    by_real = {f.real_index: f for f in features}
    if voting is not None and voting[1] == 1:
        voting = None
    if voting is not None:
        assert voting[2] > 0 and streams is None and mono is None and constraints is None and sampler is None
        voting = (voting[0], voting[1], min(voting[2], len(features)))
    before = sampler.rnd.draws if sampler is not None else 0
    if sampler is not None:
        assert used is None
        used = sampler.by_tree()
    used = set(by_real) if used is None else set(used)
    sets = I.sets_of(constraints if constraints is not None else [list(by_real)], max(by_real) + 1)
    ranks = 1 if voting is None else voting[1]
    n = len(g)
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags=[{fi: fi in used for fi in by_real} for _ in range(ranks)], bounds=NO_BOUNDS, depth=0, mask=I.ALL, branch=())]
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
            rnd, samples, voted = [], [], []
            for l in new_leaves:
                L = leaves[l]
                if voting is None:
                    scans = scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"][0], p, streams, mono,
                                      penalty, L["bounds"], L["depth"])
                    for fi, s in scans.items():
                        L["flags"][0][fi] = s.splittable
                else:
                    v, scans = _vote(bins, g, h, L, features, p, voting)
                    voted.append(v)
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
            if voting is not None:
                T["voted"].append((voted[0], voted[1] if len(voted) > 1 else None))
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
        left_out = M.constrained_output(s.left_g, s.left_h, p, s.l2, lo, hi)
        right_out = M.constrained_output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, p, s.l2, lo, hi)
        lb, rb = M.child_bounds(L["bounds"], 0 if mono is None or s.is_cat else mono[s.feature], s.is_cat, left_out, right_out)
        mask, branch = L["mask"] & sets[s.feature], L["branch"] + (s.feature,)
        lrows, rrows = L["rows"][left], L["rows"][~left]
        lcount, rcount = (len(lrows), len(rrows)) if voting is None and not estimated_counts else (s.left_count, L["count"] - s.left_count)
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
        flags = [dict(fl) for fl in L["flags"]]
        R = dict(rows=rrows, sum_g=L["sum_g"] - s.left_g, sum_h=sum_h2 - s.left_h - ref.K_EPS, count=rcount, best=None,
                 value=0.0 if math.isnan(right_out) else right_out, weight=sum_h2 - s.left_h - ref.K_EPS, flags=[dict(fl) for fl in flags],
                 bounds=rb, depth=L["depth"] + 1, mask=mask, branch=branch)
        L.update(rows=lrows, sum_g=s.left_g, sum_h=s.left_h - ref.K_EPS, count=lcount, best=None,
                 value=0.0 if math.isnan(left_out) else left_out, weight=s.left_h - ref.K_EPS, flags=flags, bounds=lb, depth=L["depth"] + 1,
                 mask=mask, branch=branch)
        leaves.append(R)
        parent_of[pick] = node
        parent_of.append(node)
        new_leaves = [pick, nl]
    T["num_leaves"] = len(leaves)
    T["leaf_value"] = [L["value"] if abs(L["value"]) > ref.K_ZERO else 0.0 for L in leaves]
    T["leaf_weight"] = [L["weight"] for L in leaves]
    T["leaf_count"] = [L["count"] for L in leaves]
    T["leaf_rows"] = [L["rows"] for L in leaves]
    T["internal_value"] = [v if abs(v) > ref.K_ZERO else 0.0 for v in T["internal_value"]]
    T["bounds"] = [L["bounds"] for L in leaves]
    T["masks"] = [L["mask"] for L in leaves]
    T["branches"] = [L["branch"] for L in leaves]
    T["draws"] = sampler.rnd.draws - before if sampler is not None else 0
    return T
