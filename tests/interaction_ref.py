"""NumPy restatement of LightGBM 3.2's interaction constraints (`interaction_constraints`) on top of split_scan_ref.py, and of
extra_trees_ref.py and monotone_ref.py for the combined cases, used to pin the engine's pick step (d_pick_block) and the round
controller's leaf set masks tree by tree.

Restated from LightGBM 3.2 (ColSampler::GetByNode, Tree::branch_features, SerialTreeLearner::ComputeBestSplitForFeature); not checked
against the native library:
- `constraints` is a list of sets of real feature indices.  A leaf's branch is the real split features on its path from the root.  A set
  is compatible with the leaf when it holds every branch feature (every set is compatible with the root); the features allowed at the
  leaf are the branch features and the union of the compatible sets (`allowed_by_branch`).
- The scans run as without constraints, for every feature the tree's feature_fraction sample holds: the same is_splittable flag updates
  and the same extra_trees draws.  Only the leaf's best split is taken over the allowed features alone (`best_of_leaf`).

The engine keeps one bit mask per leaf instead (`allowed_by_mask`): sets_of[f] has bit s set when set s holds f, the root's mask has
every bit, a split on f gives both children parent & sets_of[f], and f is allowed where sets_of[f] & mask != 0.  The restatement grows
trees with the masks; test_interaction_reference_cpu.py checks that the two forms agree."""
import math

import numpy as np

import extra_trees_ref as X3
import monotone_ref as M
import split_scan_ref as ref

ALL = (1 << 64) - 1      # the root's mask: every set


def allowed_by_branch(constraints, branch, features):
    """GetByNode's rule: the real indices among `features` allowed at a leaf whose path splits on `branch`"""
    allowed = set(branch)
    for c in constraints:
        if all(f in c for f in branch):
            allowed |= set(c)
    return {f for f in features if f in allowed}


def sets_of(constraints, nf):
    """[nf] per real feature, bit s set when set s holds it"""
    out = [0] * nf
    for s, c in enumerate(constraints):
        for f in c:
            out[f] |= 1 << s
    return out


def allowed_by_mask(sets, mask, features):
    return {f for f in features if sets[f] & mask}


def best_of_leaf(scans, sets, mask):
    """split_scan_ref.best_of_leaf over the features the leaf's mask allows"""
    return ref.best_of_leaf({fi: s for fi, s in scans.items() if sets[fi] & mask})


def grow_tree(bins, g, h, features, p, num_leaves, constraints, extra_trees=False, extra_seed=6, streams=None, used=None, mono=None,
              penalty=0.0):
    """split_scan_ref.grow_tree under interaction constraints (non-empty), with extra_trees as extra_trees_ref.grow_tree's and, with a
    `mono` list, monotone constraints as monotone_ref.grow_tree's.  `used`: the real indices the tree's feature_fraction sample holds
    (None: every feature).  T["masks"]: every leaf's final mask; T["branches"]: every leaf's split features from the root;
    T["scan_masks"]: per round, the mask of each leaf scanned, in T["rounds"]'s order."""
    features = sorted(features, key=lambda f: f.real_index)
    if extra_trees and streams is None:
        streams = X3.Streams(features, extra_seed)
    if not extra_trees:
        streams = None
    used = {f.real_index for f in features} if used is None else set(used)
    sets = sets_of(constraints, max(f.real_index for f in features) + 1)
    n = len(g)
    by_real = {f.real_index: f for f in features}
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags={f.real_index: f.real_index in used for f in features}, bounds=(-math.inf, math.inf), depth=0, mask=ALL, branch=())]
    T = dict(split_feature=[], threshold_bin=[], default_left=[], is_cat=[], cat_bins=[], split_gain=[], left_child=[], right_child=[],
             internal_value=[], internal_weight=[], internal_count=[])
    parent_of = [-1]
    rounds, picks, scan_masks = [], [], []
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
                if mono is not None:
                    scans = M.scan_leaf(bins, g, h, L["rows"], L, features, p, mono, penalty, streams, used)
                elif streams is not None:
                    scans = X3.scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"], p, streams, used)
                else:
                    scans = ref.scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"], p)
                for fi, s in scans.items():
                    L["flags"][fi] = s.splittable
                L["best"] = best_of_leaf(scans, sets, L["mask"])
                rnd.append((l, L, scans))
            rounds.append(rnd)
            scan_masks.append([leaves[l]["mask"] for l, _, _ in rnd])
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
        if mono is not None:
            left_out = M.constrained_output(s.left_g, s.left_h, p, s.l2, lo, hi)
            right_out = M.constrained_output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, p, s.l2, lo, hi)
            lb, rb = M.child_bounds(L["bounds"], 0 if s.is_cat else mono[s.feature], s.is_cat, left_out, right_out)
        else:
            left_out = ref.calc_output(s.left_g, s.left_h, p, s.l2)
            right_out = ref.calc_output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, p, s.l2)
            lb = rb = L["bounds"]
        mask, branch = L["mask"] & sets[s.feature], L["branch"] + (s.feature,)
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
                 depth=L["depth"] + 1, mask=mask, branch=branch)
        L.update(rows=lrows, sum_g=s.left_g, sum_h=s.left_h - ref.K_EPS, count=len(lrows), best=None,
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
    T["internal_value"] = [v if abs(v) > ref.K_ZERO else 0.0 for v in T["internal_value"]]
    T["masks"] = [L["mask"] for L in leaves]
    T["branches"] = [L["branch"] for L in leaves]
    T["scan_masks"] = scan_masks
    T["rounds"], T["picks"], T["scanned_counts"] = rounds, picks, []
    return T


def leaf_paths(t):
    """the split features on every root-to-leaf path of a parsed model tree (modeltext.parse_model)"""
    if t["num_leaves"] <= 1:
        return [[]]
    out = []

    def walk(node, path):
        path = path + [int(t["split_feature"][node])]
        for child in (int(t["left_child"][node]), int(t["right_child"][node])):
            if child < 0:
                out.append(path)
            else:
                walk(child, path)
    walk(0, [])
    return out
