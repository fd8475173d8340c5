"""NumPy restatement of LightGBM 3.2's tree walks, the known answer for every predictor of the engine.

`decide` is Tree::NumericalDecision / Tree::CategoricalDecision on raw feature values and `decide_bin` is NumericalDecisionInner /
CategoricalDecisionInner on the bins of a dataset.  Trees are the dicts of `mmlspark_b200.modeltext.parse_model`.

The raw walk is written for x86, the platform LightGBM's JVM bindings ship for: `static_cast<int>(double)` compiles to cvttsd2si,
which truncates toward zero and gives INT_MIN (0x80000000) for NaN, for +-inf and for any value whose truncation lies outside the
int32 range.  CategoricalDecision converts before it looks at NaN:

    int int_fval = static_cast<int>(fval);
    if (int_fval < 0) return right;
    else if (std::isnan(fval)) { if (missing_type == NaN) return right; int_fval = 0; }

so on x86 a categorical NaN goes right whatever the node's missing type, and the "NaN -> category 0" branch never runs.  This is
reasoned from the source and the x86 conversion rule, not measured against a LightGBM build.

kZeroThreshold is the engine's 1e-35.  LightGBM's meta.h may spell it as the float literal 1e-35f (1.0000000180025095e-35 as a double);
that is not settled here, and the tests use the engine's constant.
"""
import itertools
import math

import numpy as np

K_ZERO_THRESHOLD = 1e-35
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
MISSING_NONE, MISSING_ZERO, MISSING_NAN = 0, 1, 2


def x86_int(v):
    """static_cast<int>(double v) on x86 (cvttsd2si): truncation toward zero, INT_MIN when the result is not an int32"""
    v = float(v)
    if math.isnan(v) or math.isinf(v):
        return INT_MIN
    t = math.trunc(v)
    return t if INT_MIN <= t <= INT_MAX else INT_MIN


def missing_type(tree, node):
    return (int(tree["decision_type"][node]) >> 2) & 3


def default_left(tree, node):
    return bool(int(tree["decision_type"][node]) & 2)


def is_categorical(tree, node):
    return bool(int(tree["decision_type"][node]) & 1)


def cat_words(tree, node):
    """the bitset of categories that go left at a categorical node: threshold = index into cat_boundaries"""
    k = int(tree["threshold"][node])
    cb = tree["cat_boundaries"]
    return [int(w) for w in tree["cat_threshold"][int(cb[k]):int(cb[k + 1])]]


def in_bitset(words, pos):
    """Common::FindInBitset: a position past the last word is not in the set"""
    return 0 <= pos and (pos >> 5) < len(words) and bool((words[pos >> 5] >> (pos & 31)) & 1)


def _child(tree, node, left):
    return int(tree["left_child"][node]) if left else int(tree["right_child"][node])


def decide(tree, node, x):
    """child of `node` for the raw value x of its split feature"""
    v = float(x)
    mt = missing_type(tree, node)
    if is_categorical(tree, node):
        iv = x86_int(v)
        if iv < 0:                                  # NaN, +-inf, negatives and values past int32 end here on x86
            return _child(tree, node, False)
        if math.isnan(v):                           # unreachable on x86: kept to show where LightGBM's text differs from what runs
            if mt == MISSING_NAN:
                return _child(tree, node, False)
            iv = 0
        return _child(tree, node, in_bitset(cat_words(tree, node), iv))
    if math.isnan(v) and mt != MISSING_NAN:
        v = 0.0
    if (mt == MISSING_ZERO and abs(v) <= K_ZERO_THRESHOLD) or (mt == MISSING_NAN and math.isnan(v)):
        return _child(tree, node, default_left(tree, node))
    return _child(tree, node, v <= float(tree["threshold"][node]))


def feature_meta(num_bin, default_bin, upper, bin_to_cat=None):
    """what decide_bin needs of one feature of a dataset: its bin count, the bin of 0.0, the upper bound of every bin and, for a
    categorical feature, the category of every bin (bin 0: NaN, negative, rare and unseen categories)"""
    return dict(num_bin=int(num_bin), default_bin=int(default_bin), upper=np.asarray(upper, dtype=np.float64),
                bin_to_cat=None if bin_to_cat is None else [int(c) for c in bin_to_cat])


def avoid_inf(t):
    """the model-text threshold of a bin bound (Tree::Split's AvoidInf)"""
    if math.isnan(t):
        return 0.0
    return 1e300 if t >= 1e300 else -1e300 if t <= -1e300 else t


def threshold_in_bin(tree, node, meta):
    """the bin a numerical node splits after: the one bin whose bound becomes the node's threshold in the model text"""
    thr = float(tree["threshold"][node])
    if "bins_of_threshold" not in meta:
        meta["bins_of_threshold"] = {}
        for b, u in enumerate(meta["upper"]):
            if not math.isnan(u):                   # the NaN bin's bound is no threshold
                meta["bins_of_threshold"].setdefault(avoid_inf(float(u)), []).append(b)
    hits = meta["bins_of_threshold"].get(thr, [])
    assert len(hits) == 1, "threshold %r is the bound of bins %s" % (thr, hits)
    return hits[0]


def decide_bin(tree, node, b, meta):
    """child of `node` for bin b of its split feature; meta = feature_meta of that feature in the dataset the bins come from"""
    b = int(b)
    if is_categorical(tree, node):                  # the bin bitset holds the bins of the left categories; bin 0 is never in it
        cats = meta["bin_to_cat"]
        return _child(tree, node, b != 0 and in_bitset(cat_words(tree, node), cats[b]))
    mt = missing_type(tree, node)
    if (mt == MISSING_ZERO and b == meta["default_bin"]) or (mt == MISSING_NAN and b == meta["num_bin"] - 1):
        return _child(tree, node, default_left(tree, node))
    return _child(tree, node, b <= threshold_in_bin(tree, node, meta))


def leaf_index(tree, row, step=None):
    """leaf a row reaches; step(tree, node, value) defaults to decide on raw values"""
    if int(tree["num_leaves"]) <= 1:
        return 0
    step = step or decide
    node = 0
    while node >= 0:
        node = step(tree, node, row[int(tree["split_feature"][node])])
    return ~node


def bin_leaf_index(tree, bins_row, metas):
    """leaf a row of bins reaches; metas[f] = feature_meta of real feature f"""
    return leaf_index(tree, bins_row, lambda t, n, b: decide_bin(t, n, b, metas[int(t["split_feature"][n])]))


def iteration_range(num_trees, K, start_iteration=0, num_iteration=-1):
    """[t0, t1) of the trees a prediction walks (HostModel::IterRange)"""
    total = num_trees // K
    s = min(max(start_iteration, 0), total)
    e = min(s + num_iteration, total) if num_iteration > 0 else total
    return s * K, e * K


def leaf_indices(trees, X, K=1, start_iteration=0, num_iteration=-1):
    """[rows][trees of the range] leaf index per tree"""
    t0, t1 = iteration_range(len(trees), K, start_iteration, num_iteration)
    return np.array([[leaf_index(trees[t], x) for t in range(t0, t1)] for x in X], dtype=np.float64).reshape(len(X), t1 - t0)


def scores_from_leaves(trees, leaves, K=1, start_iteration=0, num_iteration=-1, average=False):
    """[rows][K] raw scores: fp64 sums in model order, tree t to class t mod K, from 0.0; divided by the iterations for an averaged
    (rf) model.  leaves = [rows][trees of the range] as leaf_indices gives."""
    t0, t1 = iteration_range(len(trees), K, start_iteration, num_iteration)
    out = np.zeros((len(leaves), K))
    for i, row in enumerate(leaves):
        acc = [0.0] * K
        for t in range(t0, t1):
            acc[t % K] += float(trees[t]["leaf_value"][int(row[t - t0])])
        out[i] = acc
    if average and t1 > t0:
        out /= (t1 - t0) // K
    return out


def raw_scores(trees, X, K=1, start_iteration=0, num_iteration=-1, average=False):
    return scores_from_leaves(trees, leaf_indices(trees, X, K, start_iteration, num_iteration), K, start_iteration, num_iteration, average)


def brute_force_shap(tree, x):
    """Shapley values of one tree by the DEFINITION: v(S) = E[f(x) | x_S] with the features outside S integrated out along the tree by
    the training cover of the children (the path-dependent expectation TreeSHAP computes), phi_i = sum over subsets of the weighted
    marginal contributions.  Exponential in the number of features a tree uses — a known-answer generator, not an algorithm.
    Returns ({feature: phi}, expected value)."""
    if int(tree["num_leaves"]) <= 1:
        return {}, float(tree["leaf_value"][0])
    sf = [int(v) for v in tree["split_feature"]]
    lc, rc = [int(v) for v in tree["left_child"]], [int(v) for v in tree["right_child"]]
    lv = [float(v) for v in tree["leaf_value"]]
    lcnt, icnt = [float(v) for v in tree["leaf_count"]], [float(v) for v in tree["internal_count"]]
    hot = [decide(tree, n, x[sf[n]]) for n in range(len(sf))]

    def cover(n):
        return icnt[n] if n >= 0 else lcnt[~n]

    def ev(n, S):
        if n < 0:
            return lv[~n]
        if sf[n] in S:
            return ev(hot[n], S)
        return (cover(lc[n]) * ev(lc[n], S) + cover(rc[n]) * ev(rc[n], S)) / cover(n)

    feats = sorted(set(sf))
    M = len(feats)
    phi = {f: 0.0 for f in feats}
    for i in feats:
        others = [f for f in feats if f != i]
        for k in range(len(others) + 1):
            wgt = math.factorial(k) * math.factorial(M - k - 1) / math.factorial(M)
            for S in itertools.combinations(others, k):
                S = set(S)
                phi[i] += wgt * (ev(0, S | {i}) - ev(0, S))
    return phi, ev(0, set())


def contributions(trees, x, num_feature, K=1, start_iteration=0, num_iteration=-1):
    """[K * (num_feature + 1)] brute-force contributions of one row, LightGBM's layout: per class, one per feature then the expected value"""
    t0, t1 = iteration_range(len(trees), K, start_iteration, num_iteration)
    out = np.zeros((K, num_feature + 1))
    for t in range(t0, t1):
        phi, e = brute_force_shap(trees[t], x)
        for f, v in phi.items():
            out[t % K, f] += v
        out[t % K, num_feature] += e
    return out.ravel()


# ---------------------------------------------------------------- rows at the edges of a forest's decisions
TINY = 1e-35
SUBNORMAL = 5e-324
CATEGORY_EDGES = (np.nan, -1.0, -0.5, -0.0, 0.0, 0.5, 0.99, 31.9, 32.0, float(INT_MAX), 2.0 ** 31, 3e9, -3e9, np.inf, -np.inf)


def numeric_edges(thresholds):
    """every threshold, one ulp either side, +-0, +-1e-35 and one ulp either side of each, the smallest subnormal, +-1e300, +-1e308,
    +-inf and NaN"""
    vals = [0.0, -0.0, SUBNORMAL, -SUBNORMAL, 1e300, -1e300, 1e308, -1e308, np.inf, -np.inf, np.nan]
    for t in list(thresholds) + [TINY, -TINY]:
        t = float(t)
        vals += [t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)]
    return vals


def categorical_edges(trees, f):
    """CATEGORY_EDGES, every left category of feature f, and the first category past the longest bitset of its nodes"""
    vals = list(CATEGORY_EDGES)
    longest = 0
    for t in trees:
        for n in range(int(t["num_leaves"]) - 1):
            if int(t["split_feature"][n]) == f and is_categorical(t, n):
                w = cat_words(t, n)
                longest = max(longest, len(w))
                vals += [float(c) for c in range(32 * len(w)) if in_bitset(w, c)]
    vals.append(float(32 * longest))
    return vals


def edge_values(trees, f):
    """values of feature f that sit on an edge of some node splitting on it"""
    thr, cat = [], False
    for t in trees:
        for n in range(int(t["num_leaves"]) - 1):
            if int(t["split_feature"][n]) == f:
                if is_categorical(t, n):
                    cat = True
                else:
                    thr.append(float(t["threshold"][n]))
    vals = numeric_edges(sorted(set(thr)))
    if cat:
        vals += categorical_edges(trees, f)
    return vals


def edge_rows(trees, num_feature, base_rows):
    """every base row with one feature set to each of its edge values: each node meets every edge of its feature on several paths"""
    out = [np.asarray(b, dtype=np.float64) for b in base_rows]
    for f in range(num_feature):
        for v in edge_values(trees, f):
            for b in base_rows:
                r = np.array(b, dtype=np.float64)
                r[f] = v
                out.append(r)
    return np.array(out)


def categorical_features(trees):
    return sorted({int(t["split_feature"][n]) for t in trees for n in range(int(t["num_leaves"]) - 1) if is_categorical(t, n)})


# ---------------------------------------------------------------- a hand-written forest with every kind of node
def N(f, thr, dt, left, right):
    """numerical node: feature, threshold, decision_type (missing type << 2 | default_left << 1), subtrees or leaf values"""
    return ("num", f, float(thr), dt, left, right)


def C(f, cats, dt, left, right):
    """categorical node: feature, categories that go left, decision_type (missing type << 2 | 1)"""
    return ("cat", f, list(cats), dt, left, right)


# 6 features: 0-3 numerical, 4 and 5 categorical.  K = 3 classes, 3 iterations; tree 3 is a stump.  Numerical nodes of missing type
# None (dt 0/2), Zero (4/6) and NaN (8/10) with both default directions; thresholds at +-1e-35, 0, +-1e300 and ordinary values;
# categorical nodes of missing type None (1) and NaN (9) with category 0 in and out of the left set, bitsets of 1 to 3 words with left
# categories at 0, 31, 32, 63, 64 and 95.
HAND_TREES = [
    N(0, 0.0, 0, N(1, 1e-35, 4, 0.5, -0.25), N(1, -1e-35, 6, 1.25, -2.0)),
    C(4, [0, 3, 7], 1, N(2, -1e300, 8, 0.75, -0.125), C(4, [1, 2, 31], 1, 2.5, -1.5)),
    C(5, [31, 32, 63, 64, 95], 9, N(2, 1e300, 10, 0.3, -0.7), C(5, [0, 32], 9, 1.1, -0.9)),
    0.25,
    N(3, 0.5, 2, N(0, -2.25, 10, 0.6, -0.4), N(3, 1e300, 0, 1.7, -1.3)),
    N(0, 1e-35, 0, N(1, 0.0, 4, 0.2, -0.2), N(2, 0.0, 8, 0.9, N(3, -1e-35, 6, -0.6, 0.45))),
    C(4, [95], 1, 0.35, N(1, -1e300, 6, -0.15, C(5, [0], 9, 0.55, -0.85))),
    N(1, 1e300, 2, N(3, -1e-35, 8, 0.05, -0.95), C(4, [0, 64], 1, 1.45, -1.05)),
    C(5, [0], 9, 0.65, N(3, 1e-35, 6, -0.35, N(0, -1e-35, 2, 0.15, -1.15))),
]
HAND_NUM_FEATURE = 6
HAND_K = 3
HAND_BASE_ROWS = [
    [0.0, 0.0, 0.0, 0.0, 0.0, 0.0],
    [1.5, -0.3, np.nan, 0.7, 3.0, 32.0],
    [-3.0, 2e-35, 1e301, -1.0, 7.0, 95.0],
    [np.nan, np.nan, -2.0, 1e300, 64.0, 0.0],
]


def _tree_text(spec, t):
    if not isinstance(spec, tuple):
        return "num_leaves=1\nnum_cat=0\nleaf_value=%r\nis_linear=0\nshrinkage=1\n" % float(spec)
    nodes, leaves, cats = [], [], []

    def walk(s):
        if not isinstance(s, tuple):
            leaves.append(float(s))
            return ~(len(leaves) - 1)
        i = len(nodes)
        nodes.append(None)
        kind, f, thr, dt, l, r = s
        if kind == "cat":
            words = [0] * (max(thr) // 32 + 1)
            for c in thr:
                words[c >> 5] |= 1 << (c & 31)
            thr = len(cats)
            cats.append(words)
        nodes[i] = [f, thr, dt, walk(l), walk(r)]
        return i
    walk(spec)
    lcount = [3 + 2 * i + (t % 3) for i in range(len(leaves))]      # uneven covers, so every Shapley weight matters

    def count(n):
        return lcount[~n] if n < 0 else count(nodes[n][3]) + count(nodes[n][4])
    icount = [count(i) for i in range(len(nodes))]

    def value(n):
        return leaves[~n] if n < 0 else (count(nodes[n][3]) * value(nodes[n][3]) + count(nodes[n][4]) * value(nodes[n][4])) / count(n)
    bounds = [0]
    for w in cats:
        bounds.append(bounds[-1] + len(w))

    def j(v):
        return " ".join(repr(x) if isinstance(x, float) else str(x) for x in v)
    lines = ["num_leaves=%d" % len(leaves), "num_cat=%d" % len(cats),
             "split_feature=" + j([n[0] for n in nodes]), "split_gain=" + j([1.0] * len(nodes)),
             "threshold=" + j([float(n[1]) for n in nodes]), "decision_type=" + j([n[2] for n in nodes]),
             "left_child=" + j([n[3] for n in nodes]), "right_child=" + j([n[4] for n in nodes]),
             "leaf_value=" + j(leaves), "leaf_weight=" + j([float(c) for c in lcount]), "leaf_count=" + j(lcount),
             "internal_value=" + j([value(i) for i in range(len(nodes))]), "internal_weight=" + j([float(c) for c in icount]),
             "internal_count=" + j(icount)]
    if cats:
        lines += ["cat_boundaries=" + j(bounds), "cat_threshold=" + j([w for ws in cats for w in ws])]
    return "\n".join(lines + ["is_linear=0", "shrinkage=1"]) + "\n"


def hand_forest_text(specs=HAND_TREES, num_feature=HAND_NUM_FEATURE, K=HAND_K):
    """LightGBM model text v3 of the trees in `specs`, written as a LightGBM-trained multiclass model arrives"""
    cat = {s[1] for spec in specs for s in _nodes_of(spec) if s[0] == "cat"}
    infos = ["0:1:2:3" if f in cat else "[-1e+308:1e+308]" for f in range(num_feature)]
    head = ["tree", "version=v3", "num_class=%d" % K, "num_tree_per_iteration=%d" % K, "label_index=0", "max_feature_idx=%d" % (num_feature - 1),
            "objective=" + ("multiclass num_class:%d" % K if K > 1 else "regression"), "feature_names=" + " ".join("f%d" % f for f in range(num_feature)),
            "feature_infos=" + " ".join(infos), ""]
    body = "".join("Tree=%d\n%s\n" % (t, _tree_text(s, t)) for t, s in enumerate(specs))
    return "\n".join(head) + body + "end of trees\n"


def _nodes_of(spec):
    if isinstance(spec, tuple):
        yield spec
        yield from _nodes_of(spec[4])
        yield from _nodes_of(spec[5])
