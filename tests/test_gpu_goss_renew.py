"""The GOSS sample (k_goss_draw), the bagging draws (k_bag_draw: balanced fractions, bagging_freq > 1) and the percentile leaf renewal
(renew_kernel.cuh) tree by tree against the NumPy restatements goss_ref.py, tree_check.bags and renew_ref.py, each tree grown by
tree_ref.grow_tree at tree_check.compare_tree's bar.  A renewed tree's structure is compared as any other; its leaf values must equal
RoundTiny(renewed * learning_rate) (plus the init score where AddBias adds it) bit for bit, and the scores after a gbdt tree must equal
score + RoundTiny(renewed * learning_rate) on every in-bag row.  Every tree must be decided first (split_scan_ref.undecided, and no
renewal threshold within 2 ulps of a cdf value)."""
import numpy as np
import pytest

import goss_ref as G
import renew_ref as RN
import split_scan_ref as ref
import tree_check as tc
import tree_ref

pytestmark = pytest.mark.gpu


def _tiny(x):
    return x if abs(x) > ref.K_ZERO else 0.0


def _decided(T, what):
    why = ref.undecided(T)
    assert not why, "%s does not discriminate:\n%s" % (what, "\n".join(why[:10]))


# ---------------------------------------------------------------- GOSS on custom grid gradients
def _goss_grads(seed, n, K, top_rate):
    """grid (g, h) per class, class scales 1000 / 1 / 0.001 so that the float32 class sum of |g h| rounds; a block of zero gradients;
    in every other block 20 rows tied with the row at the threshold"""
    X, g, h, cats = tc.data(seed, n=n)
    rng = np.random.default_rng(seed)
    Gm = np.stack([g * 1000.0, g, np.round(g * 1024) / 1024 / 1024][:K]).astype(np.float32)
    Hm = np.stack([h, tc.grid(rng, 0.5, 1.5, n), tc.grid(rng, 0.5, 1.5, n)][:K]).astype(np.float32)
    Gm[:, 2048:3072] = 0.0
    for b in (0, 1, 3, 4):
        sl = slice(b * 1024, (b + 1) * 1024)
        tg = np.zeros(1024, np.float32)
        for k in range(K):
            tg = (tg + np.abs(Gm[k, sl] * Hm[k, sl])).astype(np.float32)
        at = b * 1024 + np.argsort(-tg, kind="stable")[max(1, int(1024 * top_rate)) - 1]
        tie = b * 1024 + rng.choice(1024, 20, replace=False)
        Gm[:, tie] = Gm[:, at][:, None]
        Hm[:, tie] = Hm[:, at][:, None]
    return X, cats, Gm, Hm


@pytest.mark.parametrize("K, top, other", [(1, 0.5, 0.25), (1, 0.2, 0.1), (3, 0.2, 0.1)])
def test_goss_custom_gradients(built, K, top, other):
    from mmlspark_b200.modeltext import parse_model
    n, iters, nl = 5 * 1024 + 3, 4, 8
    X, cats, Gm, Hm = _goss_grads(30 + K, n, K, top)
    obj = "objective=multiclass num_class=3" if K == 3 else "objective=regression"
    params = ("%s boosting=goss top_rate=%r other_rate=%r learning_rate=1 boost_from_average=false verbosity=-1 num_leaves=%d "
              "min_data_in_leaf=20 max_bin=255 %s" % (obj, top, other, nl, tc.DS))
    model = tc.run(X, Gm.reshape(-1), Hm.reshape(-1), params, iters, tc.ds_params(cats, 255), label=np.arange(n) % 3)
    feats, bins, ub, b2c = tc.dataset(X, cats, 255)
    trees = parse_model(model)["trees"]
    assert len(trees) == iters * K
    states = G.seeds(n, 3)
    sampled = 0
    for it in range(iters):
        if it < G.warm_up(1.0):
            bag, g2, h2 = np.ones(n, bool), Gm, Hm
        else:
            bag, g2, h2, states = G.draw(Gm, Hm, states, top, other)
            sampled += int((g2 != Gm).any(axis=0).sum())
        rows = np.nonzero(bag)[0]
        for k in range(K):
            T = tree_ref.grow_tree(bins[rows], tc.quantized(g2[k])[rows], tc.quantized(h2[k])[rows], feats, ref.Params(min_data_in_leaf=20), nl)
            _decided(T, "iteration %d class %d" % (it, k))
            tc.compare_tree(trees[it * K + k], T, ub, b2c)
    assert sampled > 0 and 0 < bag.sum() < n


# ---------------------------------------------------------------- GOSS and bagging on the engine's own gradients
def _no_nan(d):
    """tc.data without its NaNs: at the first iteration of binary and multiclass the gradients take two values, and a feature with
    missing values then ties its forward and reverse scans exactly, which the reference refuses to decide"""
    X, g, h, cats = d
    X = X.copy()
    X[:, 1] = np.nan_to_num(X[:, 1])
    return X, g, h, cats


def _own(X, y, cats, params, iters, lr, K, sample, rank_rows=None, port=None, num_leaves=16):
    """boost on the objective's gradients; sample(it, g, h) -> (in-bag mask, g, h) as the restatement draws them"""
    from mmlspark_b200.modeltext import parse_model
    dsp = tc.ds_params(cats, 255)
    model, grads, const_h = tc.boost(X, y, params + " " + dsp, iters, dsp, rank_rows=rank_rows, port=port, grads=True)
    feats, bins, ub, b2c = tc.dataset(X, cats, 255)
    trees = parse_model(model)["trees"]
    assert len(trees) == iters * K
    n = len(X)
    for it in range(iters):
        g, h = (a.reshape(K, n) for a in grads[it])
        bag, g, h = sample(it, g, h)
        rows = np.nonzero(bag)[0]
        for k in range(K):
            hq = np.ones(n) if const_h else tc.quantized(h[k])
            T = tree_ref.grow_tree(bins[rows], tc.quantized(g[k])[rows], hq[rows], feats, ref.Params(min_data_in_leaf=20), num_leaves,
                                   estimated_counts=rank_rows is not None)
            _decided(T, "iteration %d class %d" % (it, k))
            tc.compare_tree(trees[it * K + k], T, ub, b2c, lr)


def _goss_sampler(rank_rows, lr, top=0.2, other=0.1):
    st = {"s": [G.seeds(r, 3) for r in rank_rows]}

    def sample(it, g, h):
        if it < G.warm_up(lr):
            return np.ones(g.shape[1], bool), g, h
        bag, g2, h2, st["s"] = G.ranks_draw(g, h, st["s"], rank_rows, top, other)
        return bag, g2, h2
    return sample


@pytest.mark.parametrize("case", ["regression", "multiclass", "two_ranks"])
def test_goss_own_gradients(built, case):
    X, g, h, cats = _no_nan(tc.data(50, n=9000))
    y = -g
    K, obj, rank_rows, port = 1, "objective=regression", None, None
    if case == "multiclass":
        K, obj = 3, "objective=multiclass num_class=3"
        y = y + np.random.default_rng(50).standard_normal(len(y))      # no pure leaves, whose candidates all tie at zero gain
        y = np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])).astype(float)
    if case == "two_ranks":
        rank_rows, port = [5500, 3500], 29950
        obj += " tree_learner=data num_machines=2"
    nl = 8 if K == 3 else 16
    params = "%s boosting=goss learning_rate=0.3 boost_from_average=false num_leaves=%d min_data_in_leaf=20 verbosity=-1 metric=" % (obj, nl)
    _own(X, y, cats, params, 6, 0.3, K, _goss_sampler(rank_rows or [len(X)], 0.3), rank_rows, port, nl)


@pytest.mark.parametrize("case", ["balanced_binary", "freq3"])
def test_bagging(built, case):
    X, g, h, cats = _no_nan(tc.data(52 if case == "balanced_binary" else 51, n=9000))
    if case == "balanced_binary":
        y = (g < np.quantile(g, 0.3)).astype(float)
        params = "objective=binary pos_bagging_fraction=0.8 neg_bagging_fraction=0.35 bagging_freq=1 bagging_seed=5"
        bags = tc.bags(len(X), 6, 1.0, 5, label=y, pos=0.8, neg=0.35)
    else:
        y = -g
        params = "objective=regression bagging_fraction=0.6 bagging_freq=3 bagging_seed=5"
        bags = tc.bags(len(X), 7, 0.6, 5, freq=3)
    params += " learning_rate=0.3 boost_from_average=false num_leaves=16 min_data_in_leaf=20 verbosity=-1 metric="
    _own(X, y, cats, params, len(bags), 0.3, 1, lambda it, g, h: (bags[it], g, h))


# ---------------------------------------------------------------- leaf renewal
def _train(X, y, params, iters, dsp, weight=None, rank_rows=None, port=None):
    """per iteration the gradients and scores read before it, and the model; rank_rows: shards on one device"""
    from mmlspark_b200 import capi
    rank_rows = rank_rows or [len(X)]
    offs = np.concatenate([[0], np.cumsum(rank_rows)]).astype(int)

    def body(r):
        sl = slice(offs[r], offs[r + 1])
        full = capi.Dataset.from_mat(X, dsp)
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=full).set_field("label", np.asarray(y[sl], np.float32))
        if weight is not None:
            ds.set_field("weight", np.asarray(weight[sl], np.float32))
        b = capi.Booster(ds, params)
        try:
            seen = []
            for _ in range(iters):
                seen.append((b.get_gradients(), b.get_scores()))
                b.update_one_iter()
            seen.append((None, b.get_scores()))
            return b.save_model_to_string(), seen, b.get_info()["constant_hessian"]
        finally:
            b.free(); ds.free(); full.free()

    if len(rank_rows) == 1:
        res = [body(0)]
    else:
        res, errs = tc.on_ranks(len(rank_rows), port, body)
        assert not errs, errs
        assert all(tc.trees(r[0]) == tc.trees(res[0][0]) for r in res)
    cat = lambda j, it: np.concatenate([r[1][it][0][j] for r in res])       # noqa: E731
    grads = [(cat(0, it), cat(1, it)) for it in range(iters)]
    scores = [np.concatenate([r[1][it][1] for r in res]) for it in range(iters + 1)]
    return res[0][0], grads, scores, res[0][2]


def _percentile_grads(objective, score, y32, weight, label_weight, alpha):
    """k_grad_percentile at `score` (pinned in test_gpu_gradients.py): the first tree of a run from the average is grown at the init
    score, which the booster adds after the gradients can be read"""
    diff = score - y32.astype(np.float64)
    if objective == "quantile":
        a32 = np.float32(alpha)
        g = np.where(diff.astype(np.float32) >= 0, np.float32(1) - a32, -a32).astype(np.float32)
        g = g if weight is None else (g * weight).astype(np.float32)
    else:
        w = label_weight if objective == "mape" else weight
        g = np.sign(diff).astype(np.float32) if w is None else (np.sign(diff) * w.astype(np.float64)).astype(np.float32)
    return g, (np.ones(len(y32), np.float32) if weight is None else np.asarray(weight, np.float32))


def _zero_order_matters(leaf_rows, res, w, a):
    """the leaves whose weighted percentile changes when -0.0 residuals sort before +0.0 ones instead of tying with them"""
    hit = 0
    for rows in leaf_rows:
        r = res[rows]
        alt = np.where((r == 0) & np.signbit(r), -1e-300, r)
        v = RN.weighted_percentile(alt, w[rows], a)
        hit += (0.0 if abs(v) < 1e-200 else v) != RN.weighted_percentile(r, w[rows], a)
    return hit


def _renew_check(X, y, objective, iters, lr=0.3, num_leaves=16, min_data=20, alpha=0.9, weight=None, extra="", bfa=True, bags=None,
                 goss=None, rank_rows=None, port=None, cats=(), dsx="", block_scan_differs=False, zero_order=False):
    """train; every tree against grow_tree with the restated renewal as its leaf values.  bags: per iteration the in-bag mask; goss:
    (top_rate, other_rate); rf in `extra` renews against the constant init score; dsx: more dataset parameters.  block_scan_differs /
    zero_order: some leaf's value must change with a block-scan cdf / with -0.0 sorted before +0.0, or the case would not bite.
    Returns the leaf rows and the renewed leaf values per tree."""
    from mmlspark_b200.modeltext import parse_model
    dsp = tc.ds_params(cats, 255) + " " + dsx
    rf = "boosting=rf" in extra
    params = ("objective=%s alpha=%r learning_rate=%r num_leaves=%d min_data_in_leaf=%d boost_from_average=%s verbosity=-1 metric= "
              "%s %s" % (objective, alpha, lr, num_leaves, min_data, "true" if bfa else "false", extra, dsp))
    if rank_rows:
        params += " tree_learner=data num_machines=%d" % len(rank_rows)
    model, grads, scores, const_h = _train(X, y, params, iters, dsp, weight, rank_rows, port)
    feats, bins, ub, b2c = tc.dataset(X, cats, 255, dsx)
    trees = parse_model(model)["trees"]
    assert len(trees) == iters
    n = len(X)
    R = len(rank_rows) if rank_rows else 1
    rank_of_row = np.repeat(np.arange(R), rank_rows) if rank_rows else None
    a = RN.renew_alpha(objective, alpha)
    lw = RN.mape_weights(y, weight) if objective == "mape" else None
    rw = lw if objective == "mape" else weight
    y32 = np.asarray(y, np.float32)
    # the init score: the label percentile in float32 (BoostFromScore), dropped when |init| <= 1e-15
    init = 0.0
    if bfa:
        init = float(RN.percentile(y32, a, np.float32) if rw is None else RN.weighted_percentile(y32, rw, a, np.float32))
        init = init if abs(init) > ref.K_EPS else 0.0
        if not rf:      # the first tree's scores start at the init score
            assert np.array_equal(scores[0], np.zeros(n))
    states = [G.seeds(r, 3) for r in (rank_rows or [n])]
    out, differs, zeros = [], 0, 0
    for it in range(iters):
        before = scores[it] + (init if it == 0 and not rf else 0.0)
        if rf or (it == 0 and init != 0.0):      # rf: gradients taken once, at the init score
            g, h = _percentile_grads(objective, np.full(n, init) if rf else before, y32, weight, lw, alpha)
        else:
            g, h = grads[it]
            assert all(np.array_equal(u, v) for u, v in zip((g, h), _percentile_grads(objective, before, y32, weight, lw, alpha)))
        bag = np.ones(n, bool) if bags is None else bags[it]
        if goss is not None and it >= G.warm_up(lr):
            bag, g2, h2, states = G.ranks_draw(g[None], h[None], states, rank_rows or [n], *goss)
            g, h = g2[0], h2[0]
        rows = np.nonzero(bag)[0]
        hq = np.ones(n) if const_h and goss is None else tc.quantized(h)
        T = tree_ref.grow_tree(bins[rows], tc.quantized(g)[rows], hq[rows], feats, ref.Params(min_data_in_leaf=min_data), num_leaves,
                               estimated_counts=R > 1)
        _decided(T, "iteration %d" % it)
        leaf_rows = [rows[r] for r in T["leaf_rows"]]
        why = []
        score = init if rf else before
        renewed = RN.renew(leaf_rows, y, score, a, rw, rank_of_row, R, why)
        assert not why, "iteration %d: %s" % (it, why[:3])
        if block_scan_differs:
            differs += sum(u != v for u, v in zip(renewed, RN.renew(leaf_rows, y, score, a, rw, rank_of_row, R, scan=RN.block_scan_cdf)))
        if zero_order:
            zeros += _zero_order_matters(leaf_rows, y32.astype(np.float64) - score, rw, a)
        shrink = 1.0 if rf else lr
        bias = init if (rf or it == 0) and init != 0.0 else None
        fix = lambda v: _tiny(_tiny(v * shrink) + bias) if bias is not None else _tiny(v * shrink)       # noqa: E731
        T2 = dict(T, leaf_value=[fix(v) for v in renewed], internal_value=[fix(v) for v in T["internal_value"]])
        t = trees[it]
        tc.compare_tree(t, T2, ub, b2c)
        assert t["leaf_value"].tolist() == T2["leaf_value"], "iteration %d: leaf values %r vs renewed %r" % (it, t["leaf_value"], T2["leaf_value"])
        if not rf:
            for rr, v in zip(leaf_rows, renewed):
                want = before[rr] + _tiny(v * lr)
                assert np.array_equal(scores[it + 1][rr], want), "iteration %d: scores differ from score + RoundTiny(renewed * lr)" % it
        out.append((leaf_rows, renewed))
    assert not block_scan_differs or differs > 0, "a block-scan cdf must change some leaf value, or the case would not bite"
    assert not zero_order or zeros > 0, "the order of -0.0 and +0.0 must change some leaf value, or the case would not bite"
    return out


def _data(seed, n, ties=False):
    X, g, h, cats = tc.data(seed, n=n)
    y = -g * 4
    return X, (np.round(y) if ties else y), cats


@pytest.mark.parametrize("weighted", [False, True])
def test_renew_tied_integer_residuals(built, weighted):
    X, y, cats = _data(60, 6000, ties=True)
    w = np.random.default_rng(58).uniform(0.5, 3.0, len(X)).astype(np.float32) if weighted else None
    _renew_check(X, y, "regression_l1", 4, lr=1.0, weight=w, cats=cats)


def test_renew_signed_zero_residuals(built):
    """x0 = 0: 60 residuals of -1 (weight 1), zeros alternating +0.0 (weight 1, first in row order) and -0.0 (weight 4), 11 of +1;
    the threshold 60.5 falls in the first zero's weight, so which zero comes first (row order, as upstream's stable sort has it) decides
    the interpolation.  x0 = 1: 30 rows of +5, so that the tree splits on x0."""
    lab = [-1.0] * 60 + [0.0, -0.0] * 10 + [1.0] * 11 + [5.0] * 30
    w = np.array([1.0] * 60 + [1.0, 4.0] * 10 + [1.0] * 11 + [1.0] * 30, np.float32)
    X = np.zeros((len(lab), 1))
    X[-30:, 0] = 1.0
    out = _renew_check(X, np.array(lab), "quantile", 1, lr=1.0, num_leaves=2, min_data=5, alpha=0.5, bfa=False, weight=w,
                       dsx="min_data_in_leaf=5", zero_order=True)
    assert sorted(out[0][1]) == [-1.125, 5.0]


def test_renew_eleven_row_leaf_float32_alpha(built):
    """x0 = 2 on exactly 11 rows with distinct labels: a leaf of those 11 rows, where alpha 0.3 as float32 takes another order statistic
    than alpha 0.3 as double"""
    rng = np.random.default_rng(62)
    n = 600
    pick = rng.choice(n, 51, replace=False)
    X = np.zeros((n, 1))
    X[pick[:11], 0], X[pick[11:], 0] = 2.0, 1.0
    y = rng.standard_normal(n)
    y[pick[:11]] = 100.0 + 3.0 * rng.permutation(11)
    y[pick[11:]] = -50.0 + rng.standard_normal(40)
    out = _renew_check(X, y, "quantile", 1, lr=1.0, num_leaves=3, min_data=5, alpha=0.3, dsx="min_data_in_leaf=5")
    leaf_rows, renewed = out[0]
    at = [len(r) for r in leaf_rows].index(11)
    res = np.asarray(y, np.float32)[leaf_rows[at]].astype(np.float64) - float(RN.percentile(np.asarray(y, np.float32), RN.renew_alpha("quantile", 0.3), np.float32))
    assert renewed[at] != RN.percentile(res, 0.3)


@pytest.mark.parametrize("alpha", [0.01, 0.99])
def test_renew_small_leaves_extreme_alpha(built, alpha):
    """groups of 1, 2 and 3 rows that share every feature value and sit apart from the rest: leaves of 1-3 rows at min_data_in_leaf=1"""
    rng = np.random.default_rng(63)
    n = 400
    X = np.stack([rng.integers(0, 40, n).astype(float), rng.standard_normal(n)], axis=1)
    y = 0.05 * X[:, 0] + rng.standard_normal(n)
    start = 0
    for size, (x0, x1, lab) in zip((1, 2, 3), ((50.0, 0.0, 40.0), (60.0, 0.0, -40.0), (70.0, 0.0, 80.0))):
        X[start:start + size] = (x0, x1)
        y[start:start + size] = lab + np.arange(size)
        start += size
    out = _renew_check(X, y, "quantile", 2, num_leaves=6, min_data=1, alpha=alpha, dsx="min_data_in_leaf=1 min_data_in_bin=1")
    assert min(len(r) for r in out[0][0]) <= 3


@pytest.mark.parametrize("weights", ["narrow", "integer", "below_one", "wide"])
def test_renew_weighted(built, weights):
    """leaves above 3 * 1024 rows, so the cdf runs over several chunks with a carry; wide weights make the block scan's adds round"""
    X, y, cats = _data(64, 14000)
    rng = np.random.default_rng(64)
    w = {"narrow": 0.5 + np.round(rng.uniform(0, 1.5, len(X)) * 64) / 64, "integer": rng.integers(1, 20, len(X)),
         "below_one": rng.uniform(0.05, 0.99, len(X)), "wide": 10.0 ** rng.uniform(0, 7, len(X))}[weights].astype(np.float32)
    if weights == "wide":       # labels of both signs on both sides of every split, so that no gain is lost in the heaviest rows
        y = 2.0 * (X[:, 2] > 4) - 1.0 + rng.standard_normal(len(X))
    out = _renew_check(X, y, "regression_l1", 3, num_leaves=4, min_data=3100, weight=w, cats=cats, bfa=weights != "wide",
                       block_scan_differs=weights == "wide")
    assert max(len(r) for r in out[0][0]) > 3 * 1024


def test_renew_mape_wide_labels(built):
    X, y, cats = _data(65, 9000)
    y = np.sign(y) * 10.0 ** np.random.default_rng(65).uniform(0, 6, len(X))
    _renew_check(X, y, "mape", 3, num_leaves=8, cats=cats)


def test_renew_with_bagging(built):
    X, y, cats = _data(66, 9000)
    _renew_check(X, y, "regression_l1", 4, extra="bagging_fraction=0.6 bagging_freq=2 bagging_seed=3", bags=tc.bags(len(X), 4, 0.6, 3, freq=2),
                 cats=cats)


def test_renew_with_goss(built):
    """renewal on the GOSS sample, with the rows' own (not amplified) weights"""
    X, y, cats = _data(67, 9000)
    _renew_check(X, y, "regression_l1", 4, lr=0.5, extra="boosting=goss top_rate=0.3 other_rate=0.2", goss=(0.3, 0.2), cats=cats)


def test_renew_rf_quantile(built):
    X, y, cats = _data(68, 9000)
    _renew_check(X, y, "quantile", 3, alpha=0.7, extra="boosting=rf bagging_fraction=0.7 bagging_freq=1 bagging_seed=3",
                 bags=tc.bags(len(X), 3, 0.7, 3), cats=cats)


@pytest.mark.parametrize("weighted", [False, True])
def test_renew_two_ranks_one_empty_leaf(built, weighted):
    """rank 1 holds no row with x0 = 1, so that leaf is rank 0's percentile alone"""
    rng = np.random.default_rng(69)
    n0, n1 = 3000, 2500
    X = np.stack([np.concatenate([(rng.random(n0) < 0.3).astype(float), np.zeros(n1)]), rng.integers(0, 30, n0 + n1).astype(float)], axis=1)
    y = 10.0 * X[:, 0] - 0.1 * X[:, 1] + rng.standard_normal(n0 + n1)
    w = rng.uniform(0.5, 3, n0 + n1).astype(np.float32) if weighted else None
    out = _renew_check(X, y, "regression_l1", 2, num_leaves=2, weight=w, bfa=False, rank_rows=[n0, n1], port=29960 + 10 * weighted)
    assert any((r < n0).all() for r in out[0][0]), "one leaf must have no row on rank 1"
