"""NumPy restatement of LightGBM 3.2's forced splits (forcedsplits_filename): SerialTreeLearner::ForceSplits and its use in
SerialTreeLearner::Train, FeatureHistogram::GatherInfoForThreshold{Numerical,Categorical} and Dataset::BinThreshold.  It imports neither
mmlspark_b200 nor oracle.

- The plan: one JSON object {"feature", "threshold", "left", "right"}; a child is part of the plan only when it has both "feature" and
  "threshold".  Nodes are applied breadth-first from the root, one per split: node j splits the leaf its parent left it (the root's is
  leaf 0, a left child keeps its parent's leaf, the right child of node j gets leaf j + 1).
- Each node is evaluated on its leaf's histogram in the round that scans the leaf (the round after its parent was applied).  Numerical:
  the right side sums the bins above the threshold's bin, the NaN bin left out, and the left side is the leaf total minus it
  (default_left).  Categorical: the left side is the category's bin, which must not be 0.  Gains are the scans'; a node is valid only when
  its gain exceeds min_gain_shift.  min_data_in_leaf, min_sum_hessian_in_leaf, the feature sample and the interaction masks do not apply.
- The forced phase: in every round the normal scans run; then, while the phase lasts, the next node is split if its evaluation is valid.
  An invalid node (or one whose leaf was never scanned), the end of the plan or a full tree ends the phase, and that round picks as
  it would without a plan.

The grower below is tree_ref.grow_tree's round loop with the forced step added; it keeps the options the forced tests use: the
feature_fraction sample, extra-trees streams, interaction constraints, max_depth, the by-node sampler of bynode_ref.py and the path
smoothing of path_smooth_ref.py (scans, forced evaluations and children's outputs smoothed toward each leaf's output).  Quantised
training is the grower run on quant_ref.py's levels times their scales."""
import math
from collections import deque

import numpy as np

import extra_trees_ref as X3
import interaction_ref as I
import monotone_ref as M
import path_smooth_ref as PS
import split_scan_ref as ref
import tree_ref


def flatten(plan):
    """the plan's nodes breadth-first: dicts of feature, threshold, leaf, left and right (child node indices or -1)"""
    def in_plan(v):
        return isinstance(v, dict) and "feature" in v and "threshold" in v
    assert in_plan(plan)
    nodes, q = [], deque([(plan, -1, 0, 0)])
    while q:
        v, parent, side, leaf = q.popleft()
        j = len(nodes)
        nodes.append(dict(feature=int(v["feature"]), threshold=float(v["threshold"]), leaf=leaf, left=-1, right=-1))
        if parent >= 0:
            nodes[parent]["right" if side else "left"] = j
        if in_plan(v.get("left")):
            q.append((v["left"], j, 0, leaf))
        if in_plan(v.get("right")):
            q.append((v["right"], j, 1, j + 1))
    return nodes


def value_to_bin(v, f, ub, b2c):
    """Dataset::BinThreshold: a numerical value's bin (lower-bound search over the upper bounds, the NaN bin left out), or a category's bin
    (0 when the category has no bin of its own)"""
    if f.is_cat:
        c = int(v)
        hits = [b for b, cat in enumerate(b2c) if b > 0 and cat == c]
        return hits[0] if hits and c >= 0 else 0
    hi = f.num_bin - 1 - (1 if f.missing_type == 2 else 0)
    for b in range(hi):
        if v <= ub[b]:
            return b
    return hi


def with_bins(nodes, features, ub, b2c):
    """the nodes with each threshold's bin"""
    by_real = {f.real_index: f for f in features}
    return [dict(n, bin=value_to_bin(n["threshold"], by_real[n["feature"]], ub.get(n["feature"]), b2c.get(n["feature"]))) for n in nodes]


def evaluate(hg, hh, f, b, sum_g, sum_h_in, num_data, p, smooth=0.0, parent_output=0.0):
    """GatherInfoForThreshold of bin b on feature f's histogram (hg, hh): a split_scan_ref.Scan (gain - min_gain_shift, left sums with
    the scans' epsilon) when the node is valid, else None.  Also returns the half margins of the rebuilt counts and (gain, shift).
    smooth above kEpsilon: the gains of the smoothed scans toward parent_output (the leaf's output), with the sides' rebuilt counts."""
    sum_h = sum_h_in + 2 * ref.K_EPS
    cnt_factor = num_data / sum_h
    l2 = p.lambda_l2
    on = PS.active(smooth)
    shift = (PS.leaf_gain(sum_g, sum_h, num_data, parent_output, p, l2, smooth) if on else ref.leaf_gain(sum_g, sum_h, p, l2)) + p.min_gain_to_split
    margins = []
    ok = True
    if not f.is_cat:
        hi = f.num_bin - 1 - (1 if f.missing_type == 2 else 0)
        rg, rh, rc = 0.0, 0.0, 0
        for t in range(b + 1, hi + 1):
            rg += float(hg[t]); rh += float(hh[t])
            rc += ref.round_int(float(hh[t]) * cnt_factor)
            margins.append(ref.half_margin(float(hh[t]) * cnt_factor))
        rh += ref.K_EPS
        lc = num_data - rc
        lg, lh = sum_g - rg, sum_h - rh
    else:
        ok = 0 < b < f.num_bin
        g1, h1 = (float(hg[b]), float(hh[b])) if ok else (0.0, 0.0)
        lc = ref.round_int(h1 * cnt_factor)
        margins.append(ref.half_margin(h1 * cnt_factor))
        rc = num_data - lc
        lg, lh, rg = g1, h1 + ref.K_EPS, sum_g - g1
        rh = sum_h - lh
    if on:
        gain = PS.split_gain(lg, lh, rg, rh, lc, rc, parent_output, p, l2, smooth, -math.inf, math.inf, 0)
    else:
        gain = ref.leaf_gain(lg, lh, p, l2) + ref.leaf_gain(rg, rh, p, l2)
    if not (ok and gain > shift):
        return None, margins, (gain, shift)
    s = ref.Scan(f.real_index, shift)
    s.gain, s.splittable = gain - shift, True
    s.left_g, s.left_h, s.left_count, s.l2 = lg, lh, lc, l2
    s.is_cat = f.is_cat
    s.threshold, s.default_left = (0, False) if f.is_cat else (b, True)
    s.cat_bins = (b,) if f.is_cat else ()
    s.win = s._offer(gain, lg, lh, rg, rh, "forced")
    return s, margins, (gain, shift)


def leaf_histogram(bins, g, h, rows, f):
    col = bins[rows, f.real_index].astype(np.int64)
    return (np.bincount(col, weights=g[rows], minlength=f.num_bin), np.bincount(col, weights=h[rows], minlength=f.num_bin))


def grow_tree(bins, g, h, features, p, num_leaves, nodes, *, used=None, streams=None, constraints=None, max_depth=-1, sampler=None,
              smooth=0.0):
    """One tree with the forced phase.  nodes: with_bins(flatten(plan), ...).  Returns tree_ref.grow_tree's arrays, rounds and picks
    (normal picks only) and: forced = the plan nodes applied, in order; evals = per plan node, (scan or None, margins, (gain, shift)) for
    the nodes that were evaluated; phase_end = why the phase ended ('invalid', 'unscanned', 'plan', 'full' or None)."""
    features = sorted(features, key=lambda f: f.real_index)
    by_real = {f.real_index: f for f in features}
    if sampler is not None:
        assert used is None
        used = sampler.by_tree()
    used = set(by_real) if used is None else set(used)
    sets = I.sets_of(constraints if constraints is not None else [list(by_real)], max(by_real) + 1)
    n = len(g)
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags={fi: fi in used for fi in by_real}, depth=0, mask=I.ALL)]
    leaves[0]["output"] = PS.root_output(leaves[0]["sum_g"], leaves[0]["sum_h"], p)
    T = dict(split_feature=[], threshold_bin=[], default_left=[], is_cat=[], cat_bins=[], split_gain=[], left_child=[], right_child=[],
             internal_value=[], internal_weight=[], internal_count=[], rounds=[], picks=[], forced=[], evals={}, phase_end=None)
    parent_of = [-1]
    new_leaves = [0]
    forced_next = 0 if nodes else -1
    while True:
        counts = [leaves[l]["count"] for l in new_leaves]
        go = len(leaves) < num_leaves and not all(c < p.min_data_in_leaf * 2 for c in counts)
        if go and max_depth > 0 and leaves[new_leaves[0]]["depth"] >= max_depth:
            go = False
        if go:
            if len(new_leaves) == 2 and not counts[0] < counts[1]:
                new_leaves = new_leaves[::-1]
            rnd = []
            for l in new_leaves:
                L = leaves[l]
                scans = PS.scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"], p, streams, None, 0.0,
                                     tree_ref.NO_BOUNDS, L["depth"], smooth, L["output"])
                for fi, s in scans.items():
                    L["flags"][fi] = s.splittable
                allowed = {fi: s for fi, s in scans.items() if sets[fi] & L["mask"]}
                if sampler is not None:
                    sample = sampler.by_node({fi for fi in sampler.tree if sets[fi] & L["mask"]})
                    allowed = {fi: s for fi, s in allowed.items() if fi in sample}
                L["best"] = ref.best_of_leaf(allowed)
                rnd.append((l, L, scans))
                # the plan node of this leaf and round: a child of the node applied last (node 0 in round 0)
                if forced_next >= 0:
                    kids = [0] if forced_next == 0 else [nodes[forced_next - 1]["left"], nodes[forced_next - 1]["right"]]
                    for k in kids:
                        if k >= 0 and nodes[k]["leaf"] == l:
                            f = by_real[nodes[k]["feature"]]
                            hg, hh = leaf_histogram(bins, g, h, L["rows"], f)
                            T["evals"][k] = evaluate(hg, hh, f, nodes[k]["bin"], L["sum_g"], L["sum_h"], L["count"], p, smooth, L["output"])
            T["rounds"].append(rnd)
        else:
            for l in new_leaves:
                leaves[l]["best"] = None
        if len(leaves) >= num_leaves:
            if forced_next >= 0:
                T["phase_end"] = "full" if forced_next < len(nodes) else "plan"
            break
        pick, s = None, None
        if forced_next >= 0:
            j = forced_next
            ev = T["evals"].get(j)
            if j < len(nodes) and ev is not None and ev[0] is not None:
                pick, s = nodes[j]["leaf"], ev[0]
                T["forced"].append(j)
                forced_next = j + 1
            else:
                T["phase_end"] = "plan" if j >= len(nodes) else ("invalid" if ev is not None else "unscanned")
                forced_next = -1
        if pick is None:
            T["picks"].append([(li, L["best"]) for li, L in enumerate(leaves) if L["best"] is not None])
            for li, L in enumerate(leaves):
                b = L["best"]
                if b is not None and (pick is None or ref.better_split(b.gain, b.feature, leaves[pick]["best"].gain, leaves[pick]["best"].feature)):
                    pick = li
            if pick is None or not leaves[pick]["best"].gain > 0.0:
                break
            s = leaves[pick]["best"]
        L = leaves[pick]
        f = by_real[s.feature]
        left = ref.goes_left(bins[L["rows"], f.real_index].astype(np.int64), f, s)
        sum_h2 = L["sum_h"] + 2 * ref.K_EPS
        if PS.active(smooth):      # the split's estimated counts, as the pick step has them
            left_out = PS.output(s.left_g, s.left_h, s.left_count, L["output"], p, s.l2, smooth, -math.inf, math.inf)
            right_out = PS.output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, L["count"] - s.left_count, L["output"], p, s.l2, smooth, -math.inf,
                                  math.inf)
        else:
            left_out = M.constrained_output(s.left_g, s.left_h, p, s.l2, -math.inf, math.inf)
            right_out = M.constrained_output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, p, s.l2, -math.inf, math.inf)
        mask = L["mask"] & sets[s.feature]
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
        R = dict(rows=rrows, sum_g=L["sum_g"] - s.left_g, sum_h=sum_h2 - s.left_h - ref.K_EPS, count=len(rrows), best=None,
                 value=0.0 if math.isnan(right_out) else right_out, weight=sum_h2 - s.left_h - ref.K_EPS, flags=dict(L["flags"]),
                 depth=L["depth"] + 1, mask=mask, output=right_out)
        L.update(rows=lrows, sum_g=s.left_g, sum_h=s.left_h - ref.K_EPS, count=len(lrows), best=None,
                 value=0.0 if math.isnan(left_out) else left_out, weight=s.left_h - ref.K_EPS, depth=L["depth"] + 1, mask=mask,
                 output=left_out)
        leaves.append(R)
        parent_of[pick] = node
        parent_of.append(node)
        new_leaves = [pick, nl]
    T["num_leaves"] = len(leaves)
    T["leaf_value"] = [L["value"] if abs(L["value"]) > ref.K_ZERO else 0.0 for L in leaves]
    T["internal_value"] = [v if abs(v) > ref.K_ZERO else 0.0 for v in T["internal_value"]]
    T["leaf_weight"] = [L["weight"] for L in leaves]
    T["leaf_count"] = [L["count"] for L in leaves]
    T["leaf_rows"] = [np.sort(L["rows"]) for L in leaves]
    return T


def undecided(T, rel=1e-12, count_margin=1e-9):
    """split_scan_ref.undecided, plus the forced evaluations: no rebuilt count near a .5 boundary and no gain near min_gain_shift"""
    why = ref.undecided(T, rel, count_margin)
    for k, (s, margins, (gain, shift)) in T["evals"].items():
        if any(m <= count_margin for m in margins):
            why.append("forced node %d: a rebuilt count is near a .5 boundary" % k)
        if gain != shift and abs(gain - shift) <= rel * max(abs(gain), abs(shift), 1e-300):
            why.append("forced node %d: gain %.17g within %g of min_gain_shift" % (k, gain, rel))
    return why
