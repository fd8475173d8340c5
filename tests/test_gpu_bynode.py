"""Per-node feature sampling (feature_fraction_bynode): the device sampler (d_bynode_sample), the pick step's node filter and the
ColSampler stream the host and the device share, tree by tree against the NumPy restatement in bynode_ref.py (grown by tree_ref.py) on
grid gradients and at the bar tree_check.py describes, and whole models on the engine's own gradients.  Every tree of a run is grown
from the same custom (g, h): the trees differ only by the stream's position, which carries from tree to tree."""
import numpy as np
import pytest

import bynode_ref as B
import interaction_ref as I
import split_scan_ref as ref
import tree_check as tc
import tree_ref

pytestmark = pytest.mark.gpu


def _sampled_out(Ts):
    """(tree, round, leaf) where the leaf's unrestricted best feature was not in its sample: the sample changed the leaf's choice"""
    out = []
    for k, T in enumerate(Ts):
        for r, (rnd, samples) in enumerate(zip(T["rounds"], T["node_rounds"])):
            for (_, L, scans), (_, samp) in zip(rnd, samples):
                b = ref.best_of_leaf(scans)
                if b is not None and b.feature not in samp:
                    out.append((k, r))
    return out


# ---------------------------------------------------------------- tree by tree against the restatement
@pytest.mark.parametrize("bynode", [0.5, 0.8])      # 5 features: K = 3 (Floyd's branch) and K = 4 (the selection branch)
def test_numerical_with_nan(built, bynode):
    X, g, h, cats = tc.data(1, cat=True)
    _, Ts = tc.check_run(X, g, h, cats, 12, 4, bynode=bynode, extra="min_data_per_group=20 cat_smooth=5")
    assert _sampled_out(Ts), "the samples must change some leaf's choice"


def test_categoricals(built):
    """one-hot (3) and many-vs-many (4) categoricals that the gradients follow, so both split"""
    X, _, h, cats = tc.data(2, cat=True)
    rng = np.random.default_rng(21)
    y = 0.8 * (X[:, 3] == 1) + 0.6 * (X[:, 4] % 7 < 3) + 0.1 * np.nan_to_num(X[:, 1])
    g = np.round((-y + 0.3 * rng.standard_normal(len(X))) / tc.GRID) * tc.GRID
    model, Ts = tc.check_run(X, g, h, cats, 16, 3, bynode=0.6, extra="min_data_per_group=20 cat_smooth=5")
    assert tc.split_features(model) >= {3, 4}
    assert _sampled_out(Ts)


def test_wide_features(built):
    """max_bin=511: wide numerical and wide categorical features are sampled like any other"""
    X, g, h, cats = tc.data(4, n=9000, wide=True)
    model, Ts = tc.check_run(X, g, h, cats, 12, 3, bynode=0.5, max_bin=511, extra="min_data_per_group=20 cat_smooth=5")
    assert tc.split_features(model) & {3, 5}
    assert _sampled_out(Ts)


def test_feature_fraction_carries_the_stream(built):
    """the pool is the tree's feature_fraction sample, and the by-tree draws continue after the previous tree's by-node draws"""
    X, g, h, cats = tc.data(5, cat=True)
    model, Ts = tc.check_run(X, g, h, cats, 8, 6, bynode=0.7, extra="min_data_per_group=20 cat_smooth=5", fraction=0.6)
    assert all(T["draws"] > 0 for T in Ts)
    assert len({tuple(T["split_feature"]) for T in Ts}) > 1


def test_interaction_constraints(built):
    """K = 3 of 5; the gradients follow feature 4, which is only in the set [3, 4], so the leaves below a split on it have a pool of
    2 < K, which they sample whole"""
    X, _, h, cats = tc.data(3, cat=True)
    X[:, 4] = X[:, 4] % 9
    rng = np.random.default_rng(31)
    y = 1.5 * (X[:, 4] < 4) + 0.8 * (X[:, 3] == 1) + 0.1 * np.nan_to_num(X[:, 1])
    g = np.round((-y + 0.3 * rng.standard_normal(len(X))) / tc.GRID) * tc.GRID
    cons = [[0, 1, 2, 3], [3, 4]]
    model, Ts = tc.check_run(X, g, h, cats, 12, 4, bynode=0.5, cons=cons, extra="min_data_per_group=20 cat_smooth=5")
    sets = I.sets_of(cons, X.shape[1])
    capped = [samp for T in Ts for rnd in T["node_rounds"] for mask, samp in rnd if sum(1 for f in range(5) if sets[f] & mask) < 3]
    assert capped and all(samp <= {3, 4} for samp in capped)
    assert tc.paths_inside(model, cons) == 0


def test_extra_trees_draws_of_unsampled_features(built):
    """every scanned feature draws, sampled or not; the case has a feature drawn at a leaf that did not sample it, scanned again later"""
    X, g, h, cats = tc.data(13, cat=True)
    _, Ts = tc.check_run(X, g, h, cats, 12, 4, bynode=0.5, extra="min_data_per_group=20 cat_smooth=5", extra_seed=9)
    events = [(fi, fi in samp) for T in Ts for rnd, samples in zip(T["rounds"], T["node_rounds"])
              for (_, _, scans), (_, samp) in zip(rnd, samples) for fi in sorted(scans)]
    assert any(not ok and any(f2 == fi and ok2 for f2, ok2 in events[k + 1:]) for k, (fi, ok) in enumerate(events))


def test_monotone_constraints(built):
    X, g, h, cats = tc.data(1, cat=True)
    X[:, 2] = -X[:, 2]
    tc.check_run(X, g, h, cats, 12, 3, bynode=0.6, mono=[1, 0, -1, 0, 0], extra="min_data_per_group=20 cat_smooth=5")


def test_early_stop_and_max_depth(built):
    """trees that stop early (min_gain_to_split above some gains, then max_depth) take no draws after their last round, so the trees
    after them start from the exact stream position"""
    X, g, h, cats = tc.data(7, cat=True)
    feats, bins, _, _ = tc.dataset(X, cats, 255)
    T0 = tree_ref.grow_tree(bins, g, h, feats, ref.Params(min_data_in_leaf=20), 31, sampler=B.ColSampler(feats, 1.0, 0.5))
    thr = float(np.median(T0["split_gain"]))
    _, Ts = tc.check_run(X, g, h, cats, 31, 4, bynode=0.5, extra="min_gain_to_split=%r" % thr)
    assert all(1 < T["num_leaves"] < 31 for T in Ts)
    _, Ts = tc.check_run(X, g, h, cats, 31, 4, bynode=0.8, max_depth=3)
    assert all(T["num_leaves"] <= 8 for T in Ts) and all(len(T["node_rounds"]) < T["num_leaves"] for T in Ts)


def _many(seed, n=2000, nf=320):
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 8, (n, nf)).astype(np.float64)
    y = X[:, :40] @ rng.standard_normal(40) * 0.1
    g = np.round((-y + 0.2 * rng.standard_normal(n)) / tc.GRID) * tc.GRID
    return X, g, tc.grid(rng, 0.5, 1.5, n)


@pytest.mark.parametrize("bynode", [0.5, 0.05])      # 320 features: K = 160 (selection branch) and K = 16 (Floyd's branch)
def test_more_features_than_a_block(built, bynode):
    X, g, h = _many(30)
    n, k = 320, B.get_cnt(320, bynode)
    assert B.selection_branch(n, k) == (bynode == 0.5)
    _, Ts = tc.check_run(X, g, h, [], 6, 2, bynode=bynode)
    assert _sampled_out(Ts)


# ---------------------------------------------------------------- whole models on the engine's own gradients
def _base(case, extra=""):
    obj = tc.CASES[case][0]
    return "%s num_leaves=15 learning_rate=0.3 min_data_in_leaf=20 verbosity=-1 metric= %s max_bin=255 %s" % (obj, tc.DS, extra)


def _case_data(case, n=8000):
    X, z = tc.monotone_data(n, 90)
    return X, tc.CASES[case][2](z)


@pytest.mark.parametrize("case", ["regression", "binary", "multiclass", "goss", "dart", "rf", "bagging"])
def test_boosting_modes(built, case):
    """1.0 is the model of no key; 0.5 changes the trees and repeats with its seed; another feature_fraction_seed changes them"""
    X, y = _case_data(case)
    dsp = tc.DS + " max_bin=255"
    plain = tc.boost(X, y, _base(case), 5, dsp)
    assert tc.trees(tc.boost(X, y, _base(case, "feature_fraction_bynode=1.0"), 5, dsp)) == tc.trees(plain)
    a = tc.boost(X, y, _base(case, "feature_fraction_bynode=0.5"), 5, dsp)
    assert tc.trees(a) != tc.trees(plain)
    assert tc.trees(tc.boost(X, y, _base(case, "colsample_bynode=0.5"), 5, dsp)) == tc.trees(a)
    assert tc.trees(tc.boost(X, y, _base(case, "sub_feature_bynode=0.5 feature_fraction_seed=7"), 5, dsp)) != tc.trees(a)


def test_two_ranks_on_one_device(built):
    X, y = _case_data("regression")
    dsp = tc.DS + " max_bin=255"
    params = _base("regression", "feature_fraction_bynode=0.4 feature_fraction=0.8")
    one = tc.boost(X, y, params, 5, dsp)
    two = tc.boost(X, y, params + " tree_learner=data num_machines=2", 5, dsp, rank_rows=[4000, 4000], port=29900)
    assert tc.trees(one) == tc.trees(two)


def test_two_ranks_nccl(built):
    import subprocess
    from mmlspark_b200 import capi
    out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
    if len([l for l in out.splitlines() if l.startswith("GPU ")]) < 2:
        pytest.skip("needs 2 GPUs")
    X, y = _case_data("regression")
    dsp = tc.DS + " max_bin=255"
    params = _base("regression", "feature_fraction_bynode=0.4")
    one = tc.boost(X, y, params, 5, dsp)
    rows = [4000, 4000]
    offs = [0, 4000, 8000]

    def body(r):
        sl = slice(offs[r], offs[r + 1])
        full = capi.Dataset.from_mat(X, dsp)
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=full).set_field("label", np.asarray(y[sl], np.float32))
        b = capi.Booster(ds, params + " tree_learner=data num_machines=2")
        try:
            for _ in range(5):
                b.update_one_iter()
            return b.save_model_to_string()
        finally:
            b.free(); ds.free(); full.free()

    res, errs = tc.on_ranks(len(rows), 29920, body, device_of=lambda r: r)
    assert not errs, errs
    assert tc.trees(res[0]) == tc.trees(res[1]) == tc.trees(one)


def test_bundles_equal_unbundled(built):
    rng = np.random.default_rng(9)
    n = 8000
    which = rng.integers(0, 6, n)
    X = np.zeros((n, 8))
    for j in range(6):
        on = which == j
        X[on, j] = rng.integers(1, 12, on.sum())
    X[:, 6] = rng.standard_normal(n)
    X[:, 7] = rng.integers(0, 30, n)
    g = np.round((-(X[:, 0] * 0.2 + X[:, 3] * 0.1 - X[:, 1] * 0.15 + X[:, 6]) + 0.2 * rng.standard_normal(n)) / tc.GRID) * tc.GRID
    h = tc.grid(rng, 0.5, 1.5, n)
    models = []
    for bundle in ("true", "false"):
        dsp = tc.DS + " max_bin=255 enable_bundle=" + bundle
        models.append(tc.run(X, g, h, tc.params(12, "feature_fraction_bynode=0.5 enable_bundle=" + bundle), 4, dsp))
    assert tc.trees(models[0]) == tc.trees(models[1])


def test_reset_parameter(built):
    """a reset takes effect from the next tree and continues the stream: the run equals the restatement with the sampler changed in
    place after tree 1, and a reset back to 1.0 grows the plain tree"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    X, g, h, cats = tc.data(15, cat=True)
    dsp = tc.ds_params(cats, 255)
    plan = [0.5, 0.5, 0.8, 1.0, 0.5]
    ds = capi.Dataset.from_mat(X, dsp).set_field("label", np.zeros(len(X), np.float32))
    b = capi.Booster(ds, tc.params(12, "feature_fraction_bynode=0.5 min_data_per_group=20 cat_smooth=5", cats))
    try:
        for k, f in enumerate(plan):
            if k and f != plan[k - 1]:
                b.reset_parameter("feature_fraction_bynode=%r" % f)
            b.update_one_iter_custom(g.astype(np.float32), h.astype(np.float32))
        model = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    feats, bins, ub, b2c = tc.dataset(X, cats, 255)
    p = ref.Params(min_data_in_leaf=20, min_data_per_group=20, cat_smooth=5)
    trees = parse_model(model)["trees"]
    s = B.ColSampler(feats, 1.0, 0.5)
    for k, f in enumerate(plan):
        s.bynode = f
        T = tree_ref.grow_tree(bins, g, h, feats, p, 12, sampler=s)
        assert not ref.undecided(T)
        tc.compare_tree(trees[k], T, ub, b2c)
    assert "[feature_fraction_bynode: 0.5]" in model


ERRORS = [
    ("feature_fraction_bynode=0", "feature_fraction_bynode should be in (0, 1], got 0"),
    ("feature_fraction_bynode=-0.5", "got -0.5"),
    ("feature_fraction_bynode=1.5", "got 1.5"),
    ("colsample_bynode=nan", "feature_fraction_bynode should be in (0, 1]"),
]


@pytest.mark.parametrize("opts,msg", ERRORS)
def test_create_and_reset_errors(built, opts, msg):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(7, cat=True)
    ds = capi.Dataset.from_mat(X, tc.ds_params(cats, 255)).set_field("label", np.asarray(-g, np.float32))
    try:
        with pytest.raises(Exception) as e:
            capi.Booster(ds, tc.params(8, opts, cats))
        assert msg in str(e.value), str(e.value)
        b = capi.Booster(ds, tc.params(8, "feature_fraction_bynode=0.5", cats))
        try:
            b.update_one_iter()
            before = b.save_model_to_string()
            with pytest.raises(Exception) as e:
                b.reset_parameter(opts)
            assert msg in str(e.value), str(e.value)
            assert b.save_model_to_string() == before
            b.update_one_iter()
            assert "[feature_fraction_bynode: 0.5]" in b.save_model_to_string()
        finally:
            b.free()
    finally:
        ds.free()


def test_errors_fire_on_every_rank(built):
    """each range error and the voting rejection at create on both ranks, and the voting rejection at ResetParameter"""
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(25, cat=True)
    half = len(X) // 2
    cases = [(o + " tree_learner=data num_machines=2", m) for o, m in ERRORS] + \
            [("feature_fraction_bynode=0.5 tree_learner=voting top_k=2 num_machines=2", "does not support feature_fraction_bynode")]

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ds = capi.Dataset.from_mat(X[sl], tc.ds_params(cats, 255)).set_field("label", np.asarray(-g[sl], np.float32))
        try:
            msgs = []
            for opts, _ in cases:
                with pytest.raises(Exception) as e:
                    capi.Booster(ds, tc.params(8, opts, cats))
                msgs.append(str(e.value))
            b = capi.Booster(ds, tc.params(8, "tree_learner=voting top_k=2 num_machines=2", cats))
            try:
                b.update_one_iter()
                before = b.save_model_to_string()
                with pytest.raises(Exception) as e:
                    b.reset_parameter("tree_learner=data feature_fraction_bynode=0.5")
                msgs.append(str(e.value))
                after = b.save_model_to_string()
                b.update_one_iter()
                return msgs, before == after, b.save_model_to_string()
            finally:
                b.free()
        finally:
            ds.free()

    res, errs = tc.on_ranks(2, 29940, body)
    assert not errs, errs
    for msgs, unchanged, model in res:
        for (_, want), got in zip(cases + [(None, "does not support feature_fraction_bynode")], msgs):
            assert want in got, (want, got)
        assert unchanged
        assert "[feature_fraction_bynode: 1]" in model
    assert tc.trees(res[0][2]) == tc.trees(res[1][2])


def test_model_text_round_trips(built):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(8)
    dsp = tc.ds_params(cats, 255)
    model = tc.run(X, g, h, tc.params(8, "feature_fraction_bynode=0.35", cats), 2, dsp)
    assert "[feature_fraction_bynode: 0.35]" in model
    b = capi.Booster(model_str=model)
    try:
        assert b.save_model_to_string() == model
    finally:
        b.free()
    assert "[feature_fraction_bynode: 1]" in tc.run(X, g, h, tc.params(8, "", cats), 2, dsp)


def test_estimator(built):
    """LightGBMRegressor(featureFractionByNode=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    X, z = tc.monotone_data(5000, 10)
    X = np.nan_to_num(X)
    df = Frame({"features": X, "label": z})
    est = LightGBMRegressor(featureFractionByNode=0.4, numIterations=5, numTasks=1)
    model = est.fit(df).getNativeModel()
    params = est.getTrainParams(1, df).to_string()
    assert params.endswith("feature_fraction_bynode=0.4 ")
    ds = capi.Dataset.from_mat(X, dataset_params(est.get("maxBin"), est.get("binSampleCount"), est.get("numThreads"), []))
    ds.set_field("label", z.astype(np.float32))
    b = capi.Booster(ds, params)
    try:
        for _ in range(5):
            b.update_one_iter()
        low = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    assert tc.trees(model) == tc.trees(low)
    plain = LightGBMRegressor(numIterations=5, numTasks=1).fit(df).getNativeModel()
    assert tc.trees(plain) != tc.trees(model)
