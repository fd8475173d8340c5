"""Extremely randomised trees (extra_trees, extra_seed): the scans' kExtra instantiations (k_scan, k_scan_wide) and the per-feature streams
the pick step advances, tree by tree and tree after tree, against the NumPy restatement in extra_trees_ref.py (grown by tree_ref.py), on
grid gradients and at the bar tree_check.py describes.  Every tree of a run is grown from the same custom (g, h) through
UpdateOneIterCustom: the trees differ only by the streams' state, which carries from tree to tree."""
import numpy as np
import pytest

import extra_trees_ref as X3
import split_scan_ref as ref
import tree_check as tc
import tree_ref

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- tree after tree against the restatement
@pytest.mark.parametrize("seed", [6, 11, 12345])
def test_numerical_with_nan(built, seed):
    X, g, h, cats = tc.data(1)
    _, Ts = tc.check_run(X, g, h, cats, 8, 5, extra_seed=seed)
    assert len({(tuple(T["split_feature"]), tuple(T["threshold_bin"])) for T in Ts}) > 1, "the streams must carry from tree to tree"


@pytest.mark.parametrize("seed", [6, 99])
def test_one_hot_and_many_vs_many(built, seed):
    X, g, h, cats = tc.data(2, cat=True)
    model, _ = tc.check_run(X, g, h, cats, 12, 5, extra_seed=seed, extra="min_data_per_group=20 cat_smooth=5")
    assert "cat_threshold=" in model, "the case must split on a categorical feature"


def test_feature_fraction(built):
    X, g, h, cats = tc.data(3, cat=True)
    tc.check_run(X, g, h, cats, 8, 6, extra_seed=7, extra="min_data_per_group=20 cat_smooth=5", fraction=0.6)


def test_wide_features(built):
    """max_bin=511: k_scan_wide's numerical scan and a categorical feature of 600 categories"""
    X, g, h, cats = tc.data(4, n=9000, wide=True)
    model, _ = tc.check_run(X, g, h, cats, 8, 4, extra_seed=6, max_bin=511, extra="min_data_per_group=20 cat_smooth=5")
    assert tc.split_features(model) >= {3, 5}, "the case must split on the wide numerical and the wide categorical feature"


def test_reset_parameter_restarts_the_streams(built):
    """ResetParameter re-seeds every stream (LightGBM 3.2's HistogramPool::ResetConfig): the trees after a reset repeat those after
    the booster's creation"""
    X, g, h, cats = tc.data(5)
    model, _ = tc.check_run(X, g, h, cats, 8, 4, extra_seed=6, reset=(1, "learning_rate=1"))
    trees = tc.trees(model).split("Tree=")[1:]
    assert trees[0].split("\n", 1)[1] == trees[2].split("\n", 1)[1]


# ---------------------------------------------------------------- two ranks on one device
def _two_ranks(port, device_of=lambda r: 0):
    """data-parallel on two shards with unit hessians (the reconstructed global counts are exact): the model equals the one-rank model"""
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(6, cat=True, const_h=True)
    dsp = tc.ds_params(cats, 255)
    params = tc.params(10, "extra_trees=true extra_seed=21 tree_learner=data num_machines=2 min_data_per_group=20 cat_smooth=5", cats)
    half = len(X) // 2

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ref_ds = capi.Dataset.from_mat(X, dsp)      # the bins of the whole data, as one rank would have them
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=ref_ds).set_field("label", np.zeros(half, np.float32))
        b = capi.Booster(ds, params)
        try:
            for _ in range(3):
                b.update_one_iter_custom(g[sl].astype(np.float32), h[sl].astype(np.float32))
            return b.save_model_to_string()
        finally:
            b.free(); ds.free(); ref_ds.free()

    res, errs = tc.on_ranks(2, port, body, device_of)
    assert not errs, errs
    assert tc.trees(res[0]) == tc.trees(res[1])
    single, _ = tc.check_run(X, g, h, cats, 10, 3, extra_seed=21, extra="min_data_per_group=20 cat_smooth=5")
    assert tc.trees(res[0]) == tc.trees(single)


def test_two_ranks_on_one_device(built):
    _two_ranks(29600)


def test_two_ranks_nccl(built):
    import subprocess
    out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
    if len([l for l in out.splitlines() if l.startswith("GPU ")]) < 2:
        pytest.skip("needs 2 GPUs")
    _two_ranks(29620, device_of=lambda r: r)


def test_voting_rejects_at_create(built):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(7)
    params = tc.params(8, "extra_trees=true tree_learner=voting top_k=2 num_machines=2")
    half = len(X) // 2

    def body(r):
        ds = capi.Dataset.from_mat(X[r * half:(r + 1) * half], tc.ds_params((), 255)).set_field("label", np.zeros(half, np.float32))
        try:
            with pytest.raises(Exception) as e:
                capi.Booster(ds, params)
            return str(e.value)
        finally:
            ds.free()

    res, errs = tc.on_ranks(2, 29640, body)
    assert not errs, errs
    assert all("does not support extra_trees" in m for m in res), res


# ---------------------------------------------------------------- the default stays as it was; seeds, bundles, model text
def test_baseline_seeds_and_model_text(built):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(8, cat=True)
    dsp = tc.ds_params(cats, 255)
    run = lambda extra: tc.run(X, g, h, tc.params(12, extra, cats), 3, dsp)      # noqa: E731
    plain, off = run(""), run("extra_trees=false extra_seed=9")
    assert tc.trees(plain) == tc.trees(off)
    a, a2, b = run("extra_trees=true"), run("extra_tree=true extra_seed=6"), run("extra_trees=true extra_seed=7")
    assert tc.trees(a) == tc.trees(a2)
    assert tc.trees(a) != tc.trees(plain) and tc.trees(b) != tc.trees(a)
    assert "[extra_trees: 1]" in a and "[extra_seed: 6]" in a and "[extra_seed: 7]" in b
    assert "[extra_trees: 0]" in plain and "[extra_seed: 6]" in plain
    loaded = capi.Booster(model_str=b)
    try:
        assert loaded.save_model_to_string() == b
    finally:
        loaded.free()


def test_bundles_equal_unbundled(built):
    """sparse mutually exclusive features bundle into one column; the bundle members' scans draw as the plain features' do"""
    rng = np.random.default_rng(9)
    n = 8000
    which = rng.integers(0, 6, n)
    X = np.zeros((n, 8))
    for j in range(6):
        on = which == j
        X[on, j] = rng.integers(1, 12, on.sum())
    X[:, 6] = rng.standard_normal(n)
    X[:, 7] = rng.integers(0, 30, n)
    g = np.round((-(X[:, 0] * 0.2 + X[:, 3] * 0.1 + X[:, 6]) + 0.2 * rng.standard_normal(n)) / tc.GRID) * tc.GRID
    h = tc.grid(rng, 0.5, 1.5, n)
    models = []
    for bundle in ("true", "false"):
        dsp = tc.DS + " max_bin=255 enable_bundle=" + bundle
        models.append(tc.run(X, g, h, tc.params(12, "extra_trees=true extra_seed=3 enable_bundle=" + bundle), 4, dsp))
    assert tc.trees(models[0]) == tc.trees(models[1])


def test_estimator(built):
    """LightGBMRegressor(extraTrees=True, extraSeed=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    rng = np.random.default_rng(10)
    n = 5000
    X = rng.standard_normal((n, 6))
    y = X[:, 0] + 0.5 * X[:, 1] ** 2 + 0.1 * rng.standard_normal(n)
    df = Frame({"features": X, "label": y})
    est = LightGBMRegressor(extraTrees=True, extraSeed=17, numIterations=5, numTasks=1)
    model = est.fit(df).getNativeModel()
    params = est.getTrainParams(1, df).to_string()
    assert params.endswith("extra_trees=true extra_seed=17 ")
    assert "extra_trees" not in LightGBMRegressor(numIterations=5).getTrainParams(1, df).to_string()
    ds = capi.Dataset.from_mat(X, dataset_params(est.get("maxBin"), est.get("binSampleCount"), est.get("numThreads"), []))
    ds.set_field("label", y.astype(np.float32))
    b = capi.Booster(ds, params)
    try:
        for _ in range(5):
            b.update_one_iter()
        low = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    assert tc.trees(model) == tc.trees(low)
    assert "[extra_trees: 1]" in model and "[extra_seed: 17]" in model


# ---------------------------------------------------------------- a round where only the larger leaf's many-vs-many search draws
@pytest.mark.parametrize("num_cats", [40, 600])
def test_larger_leaf_draws_after_an_empty_smaller_range(built, num_cats):
    """The root splits on a 0/1 feature (2 bins: no draw, one candidate).  In the smaller child the categorical feature holds 2
    categories (max_num_cat = 1: an empty range, no draw); in the larger one it holds `num_cats` (a draw, k_scan's or, for 600
    categories, k_scan_wide's).  The larger leaf's block must not step past a draw the smaller one never took: its prefix, and every later
    draw of the feature, would otherwise differ from the restatement's."""
    rng = np.random.default_rng(num_cats)
    n = 8000 if num_cats == 40 else 12000
    x0 = (rng.random(n) < 0.75).astype(np.float64)
    c = np.where(x0 == 1, rng.integers(0, num_cats, n), rng.integers(0, 2, n)).astype(np.float64)
    x2 = rng.standard_normal(n)
    y = 6.0 * x0 + 2.0 * (c % 2 == 0) * x0 + 0.1 * x2
    g = np.round((-y + 0.2 * rng.standard_normal(n)) / tc.GRID) * tc.GRID
    h = tc.grid(rng, 0.5, 1.5, n)
    X = np.stack([x0, c, x2], axis=1)
    cats = [1]
    extra = "min_data_per_group=20 cat_smooth=5"
    p = ref.Params(min_data_in_leaf=20, min_data_per_group=20, cat_smooth=5)
    # the premise, on the reference side: root split on feature 0, then an empty range for the smaller child, a non-empty one for the larger
    left, right = x0 == 0, x0 == 1
    for rows, want_draw in ((left, False), (right, True)):
        cb = c[rows].astype(np.int64)
        from mmlspark_b200 import capi
        ds = capi.Dataset.from_mat(X, tc.ds_params(cats, 255))
        try:
            bins = ds.get_bins16()[rows, 1].astype(np.int64)
            nb = ds.feature_info(1)["num_bin"]
        finally:
            ds.free()
        hh = np.bincount(bins, weights=h[rows], minlength=nb)
        assert (X3.categorical_range(hh, nb, h[rows].sum(), int(rows.sum()), p) > 0) == want_draw, (nb, len(set(cb)))
    model, _ = tc.check_run(X, g, h, cats, 6, 4, extra_seed=6, extra=extra)
    from mmlspark_b200.modeltext import parse_model
    trees = parse_model(model)["trees"]
    assert all(int(t["split_feature"][0]) == 0 for t in trees)
    assert any(1 in t["split_feature"].tolist() for t in trees), "the categorical feature must be split on"


# ---------------------------------------------------------------- boosting runs on the engine's own gradients
def _check_boosting(X, y, objective, K, iters, extra, cats=(), extra_seed=6, fraction=1.0, bag=None, rank_rows=None, port=None):
    """every tree of the run equals tree_ref.grow_tree on the gradients it was grown from (quantised as K3 does), over its bagged rows,
    with the feature streams carried from tree to tree (K trees per iteration share them)"""
    from mmlspark_b200.modeltext import parse_model
    lr, num_leaves = 0.3, 12
    dsp = tc.ds_params(cats, 255)
    params = ("objective=%s boost_from_average=false learning_rate=%g num_leaves=%d min_data_in_leaf=20 verbosity=-1 metric= "
              "extra_trees=true extra_seed=%d %s %s" % (objective, lr, num_leaves, extra_seed, dsp, extra))
    if rank_rows:
        params += " tree_learner=data num_machines=%d" % len(rank_rows)
    model, grads, const_h = tc.boost(X, y, params, iters, dsp, rank_rows=rank_rows, port=port, grads=True)
    feats, bins, ub, b2c = tc.dataset(X, cats, 255)
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(min_data_in_leaf=20, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS})
    trees = parse_model(model)["trees"]
    assert len(trees) == iters * K
    used = X3.feature_fraction_sets(len(feats), fraction, 2, iters * K)
    bags = tc.bags(len(X), iters, bag[0], bag[1]) if bag else None
    streams = X3.Streams(feats, extra_seed)
    for it in range(iters):
        for k in range(K):
            g = grads[it][0].reshape(K, -1)[k]
            h = grads[it][1].reshape(K, -1)[k]
            gq, hq = tc.quantized(g), (np.ones(len(h)) if const_h else tc.quantized(h))
            rows = np.arange(len(g)) if bags is None else np.nonzero(bags[it])[0]
            T = tree_ref.grow_tree(bins[rows], gq[rows], hq[rows], feats, p, num_leaves, streams=streams,
                                   used={feats[i].real_index for i in used[it * K + k]})
            tc.compare_tree(trees[it * K + k], T, ub, b2c, lr)
    return model


def test_boosting_regression_with_nan(built):
    X, g, h, cats = tc.data(20)
    y = -g
    _check_boosting(X, y, "regression", 1, 5, "")


def test_boosting_binary_categorical(built):
    X, g, h, cats = tc.data(21, cat=True)
    z = -g + 3.0 * (X[:, 4] % 2 == 0) + 2.0 * (X[:, 3] == 1)
    y = (z > np.median(z)).astype(np.float64)
    model = _check_boosting(X, y, "binary", 1, 5, "min_data_per_group=20 cat_smooth=5", cats)
    assert tc.split_features(model) >= {3, 4}, "the case must split on the one-hot and the many-vs-many feature"


def test_boosting_multiclass(built):
    X, g, h, cats = tc.data(22, cat=True)
    y = np.digitize(-g, np.quantile(-g, [1 / 3, 2 / 3])).astype(np.float64)
    _check_boosting(X, y, "multiclass", 3, 3, "num_class=3 min_data_per_group=20 cat_smooth=5", cats)


def test_boosting_bagging_feature_fraction(built):
    X, g, h, cats = tc.data(23, cat=True)
    _check_boosting(X, -g, "regression", 1, 5, "bagging_fraction=0.6 bagging_freq=1 bagging_seed=7 feature_fraction=0.7 "
                    "min_data_per_group=20 cat_smooth=5", cats, fraction=0.7, bag=(0.6, 7))


def test_boosting_two_ranks_on_one_device(built):
    """data-parallel regression (unit hessians: the reconstructed global counts are exact) on two unequal shards"""
    X, g, h, cats = tc.data(24, cat=True)
    _check_boosting(X, -g, "regression", 1, 4, "min_data_per_group=20 cat_smooth=5", cats, rank_rows=[3100, 2900], port=29660)


def test_voting_reset_parameter_rejected(built):
    """a ResetParameter that turns extra_trees on under multi-rank voting fails on every rank and changes nothing"""
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(25)
    params = tc.params(8, "tree_learner=voting top_k=2 num_machines=2 boost_from_average=false")
    half = len(X) // 2

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ds = capi.Dataset.from_mat(X[sl], tc.ds_params((), 255)).set_field("label", np.asarray(-g[sl], np.float32))
        b = capi.Booster(ds, params)
        try:
            b.update_one_iter()
            with pytest.raises(Exception) as e:
                b.reset_parameter("extra_trees=true")
            b.update_one_iter()
            return str(e.value), b.save_model_to_string()
        finally:
            b.free(); ds.free()

    res, errs = tc.on_ranks(2, 29680, body)
    assert not errs, errs
    assert all("does not support extra_trees" in m for m, _ in res), res
    assert all("[extra_trees: 0]" in t for _, t in res) and tc.trees(res[0][1]) == tc.trees(res[1][1])
