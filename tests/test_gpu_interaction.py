"""Interaction constraints (interaction_constraints): the pick step's per-leaf feature filter (d_pick_block) and the round controller's
set masks, tree by tree against the NumPy restatement in interaction_ref.py (grown by tree_ref.py) on grid gradients and at the bar
tree_check.py describes, and the trained models' paths on the engine's own gradients."""
import numpy as np
import pytest

import interaction_ref as I
import split_scan_ref as ref
import tree_check as tc
import tree_ref

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- tree by tree against the restatement
def test_numerical_with_nan_overlapping_sets(built):
    X, g, h, cats = tc.data(1)
    model, _ = tc.check_run(X, g, h, cats, 12, 3, cons=[[0, 1], [1, 2]])
    assert tc.split_features(model) >= {1, 2}


def test_categoricals(built):
    """one-hot (3) and many-vs-many (4) categoricals in one set, beside a singleton and a numerical pair; the gradients follow the two
    categoricals, so both split"""
    X, _, h, cats = tc.data(2, cat=True)
    rng = np.random.default_rng(21)
    y = 0.8 * (X[:, 3] == 1) + 0.6 * (X[:, 4] % 7 < 3) + 0.1 * np.nan_to_num(X[:, 1])
    g = np.round((-y + 0.3 * rng.standard_normal(len(X))) / tc.GRID) * tc.GRID
    model, _ = tc.check_run(X, g, h, cats, 16, 3, cons=[[3, 4], [0], [1, 2]], extra="min_data_per_group=20 cat_smooth=5")
    assert tc.split_features(model) >= {3, 4}, "the case must split on the one-hot and the many-vs-many feature"


def test_wide_features(built):
    """max_bin=511: k_scan_wide's candidates pass through the same pick, for wide numerical and wide categorical features"""
    X, g, h, cats = tc.data(4, n=9000, wide=True)
    model, _ = tc.check_run(X, g, h, cats, 12, 2, cons=[[0, 3], [1, 2, 5], [4]], max_bin=511,
                            extra="min_data_per_group=20 cat_smooth=5")
    assert tc.split_features(model) & {3, 5}


def test_feature_in_no_set_and_singletons(built):
    X, g, h, cats = tc.data(3)
    model, Ts = tc.check_run(X, g, h, cats, 12, 3, cons=[[0], [2]])
    assert 1 not in tc.split_features(model)
    assert any(len(set(b)) == 1 and len(b) > 1 for T in Ts for b in T["branches"]), "a singleton must split twice on one path"


def test_feature_fraction_without_an_allowed_feature(built):
    """feature_fraction samples two of the five features per tree; iteration 6's sample, features 1 and 2, holds no allowed feature, so
    the root has no candidate and the tree has one leaf, which the booster drops; iteration 7 trains on its own sample"""
    X, g, h, cats = tc.data(5, cat=True)
    _, Ts = tc.check_run(X, g, h, cats, 8, 8, cons=[[0, 3]], extra="min_data_per_group=20 cat_smooth=5", fraction=0.4, dropped=(6,))
    assert min(T["num_leaves"] for k, T in enumerate(Ts) if k != 6) > 1


def test_extra_trees_draws_of_disallowed_features(built):
    """every scanned feature draws, allowed or not.  The case has draws of a feature at a leaf that may not split on it followed by an
    allowed scan of the same feature, so a rule that skipped the disallowed scans would shift that later draw."""
    X, g, h, cats = tc.data(13, cat=True)
    cons = [[0, 1], [0, 2, 4], [3]]
    model, Ts = tc.check_run(X, g, h, cats, 12, 4, cons=cons, extra="min_data_per_group=20 cat_smooth=5", extra_seed=9)
    sets = I.sets_of(cons, X.shape[1])
    events = [(fi, bool(sets[fi] & m)) for T in Ts for rnd, masks in zip(T["rounds"], T["scan_masks"])
              for (_, _, scans), m in zip(rnd, masks) for fi in sorted(scans)]
    assert any(not ok and any(f2 == fi and ok2 for f2, ok2 in events[k + 1:]) for k, (fi, ok) in enumerate(events)), \
        "no disallowed draw is followed by an allowed scan of the same feature"


def test_with_monotone_constraints(built):
    X, g, h, cats = tc.data(1)
    X[:, 2] = -X[:, 2]
    tc.check_run(X, g, h, cats, 12, 3, cons=[[0, 2], [1, 2]], mono=[1, 0, -1])


def test_reset_parameter_sets_changes_and_clears(built):
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    X, g, h, cats = tc.data(15)
    dsp = tc.ds_params(cats, 255)
    plan = [None, [[0, 1]], [[1, 2], [0]], None]
    ds = capi.Dataset.from_mat(X, dsp).set_field("label", np.zeros(len(X), np.float32))
    b = capi.Booster(ds, tc.params(12, "", cats))
    try:
        for k, cons in enumerate(plan):
            if k:
                b.reset_parameter(tc.ic(cons) if cons else "interaction_constraints=")
            b.update_one_iter_custom(g.astype(np.float32), h.astype(np.float32))
        model = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    feats, bins, ub, b2c = tc.dataset(X, cats, 255)
    p = ref.Params(min_data_in_leaf=20)
    trees = parse_model(model)["trees"]
    for k, cons in enumerate(plan):
        T = tree_ref.grow_tree(bins, g, h, feats, p, 12, constraints=cons)
        assert not ref.undecided(T)
        tc.compare_tree(trees[k], T, ub, b2c)
    assert "[interaction_constraints: ]" in model
    assert set(trees[1]["split_feature"].tolist()) <= {0, 1} and 2 in trees[0]["split_feature"].tolist()


# ---------------------------------------------------------------- paths on the engine's own gradients
CONS = [[0, 1], [1, 2, 3], [4]]


@pytest.mark.parametrize("case", sorted(tc.CASES))
def test_paths_stay_inside_one_set(built, case):
    obj, K, label, n = tc.CASES[case]
    n = min(n, 20000)
    X, z = tc.monotone_data(n, 70 + len(case))
    y = label(z)
    group = [20] * (n // 20) if case == "lambdarank" else None
    dsp = tc.DS + " max_bin=255"
    base = "%s num_leaves=31 learning_rate=0.3 min_data_in_leaf=20 verbosity=-1 metric= %s" % (obj, dsp)
    model = tc.boost(X, y, base + " " + tc.ic(CONS), 6, dsp, group)
    assert tc.paths_inside(model, CONS) == 0
    plain = tc.boost(X, y, base, 6, dsp, group)
    assert tc.paths_inside(plain, CONS) > 0, "the unconstrained model must break the sets, or the check would not bite"


@pytest.mark.parametrize("extra", ["", "extra_trees=true extra_seed=4"])
def test_one_set_of_every_feature_is_unconstrained(built, extra):
    X, z = tc.monotone_data(20000, 80)
    dsp = tc.DS + " max_bin=255"
    base = "objective=regression num_leaves=31 learning_rate=0.3 verbosity=-1 metric= feature_fraction=0.8 %s %s" % (extra, dsp)
    a = tc.boost(X, z, base, 6, dsp)
    b = tc.boost(X, z, base + " " + tc.ic([[4, 3, 2, 1, 0]]), 6, dsp)
    assert tc.trees(a) == tc.trees(b)


def test_two_ranks_equal_one(built):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(6, const_h=True)
    dsp = tc.ds_params(cats, 255)
    cons = [[0, 1], [1, 2]]
    params = tc.params(10, "tree_learner=data num_machines=2 " + tc.ic(cons), cats)
    half = len(X) // 2

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ref_ds = capi.Dataset.from_mat(X, dsp)
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=ref_ds).set_field("label", np.zeros(half, np.float32))
        b = capi.Booster(ds, params)
        try:
            for _ in range(3):
                b.update_one_iter_custom(g[sl].astype(np.float32), h[sl].astype(np.float32))
            return b.save_model_to_string()
        finally:
            b.free(); ds.free(); ref_ds.free()

    res, errs = tc.on_ranks(2, 29820, body)
    assert not errs, errs
    assert tc.trees(res[0]) == tc.trees(res[1])
    single, _ = tc.check_run(X, g, h, cats, 10, 3, cons=cons)
    assert tc.trees(res[0]) == tc.trees(single)


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
    cons = [[0, 6], [1, 3, 7], [2, 4, 5]]
    models = []
    for bundle in ("true", "false"):
        dsp = tc.DS + " max_bin=255 enable_bundle=" + bundle
        models.append(tc.run(X, g, h, tc.params(12, tc.ic(cons) + " enable_bundle=" + bundle), 4, dsp))
    assert tc.trees(models[0]) == tc.trees(models[1])
    assert tc.paths_inside(models[0], cons) == 0 and tc.split_features(models[0]) & {0, 1, 3}


# ---------------------------------------------------------------- errors, model text, estimator
ERRORS = [
    ("interaction_constraints=[0,1],[5]", "feature index 5 in set 1 is outside [0, 5)"),
    ("interaction_constraints=[0,-1]", "feature index -1 in set 0 is outside [0, 5)"),
    ("interaction_constraints=0,1", "got '0,1'"),
    ("interaction_constraints=[0,1],[2", "got '[0,1],[2'"),
    ("interaction_constraints=[0,x]", "got '[0,x]'"),
    ("interaction_constraints=[0,1,]", "got '[0,1,]'"),
    ("interaction_constraints=" + ",".join("[%d]" % (i % 5) for i in range(65)), "at most 64 sets"),
]


@pytest.mark.parametrize("opts,msg", ERRORS)
def test_create_errors(built, opts, msg):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(7, cat=True)
    ds = capi.Dataset.from_mat(X, tc.ds_params(cats, 255)).set_field("label", np.asarray(-g, np.float32))
    try:
        with pytest.raises(Exception) as e:
            capi.Booster(ds, tc.params(8, opts, cats))
        assert msg in str(e.value), str(e.value)
        b = capi.Booster(ds, tc.params(8, tc.ic([[0, 1]]), cats))
        try:
            b.update_one_iter()
            before = b.save_model_to_string()
            with pytest.raises(Exception) as e:
                b.reset_parameter(opts)
            assert msg in str(e.value), str(e.value)
            assert b.save_model_to_string() == before
            b.update_one_iter()
            assert tc.paths_inside(b.save_model_to_string(), [[0, 1]]) == 0
        finally:
            b.free()
    finally:
        ds.free()


def test_errors_fire_on_every_rank(built):
    """each create-time error and the voting rejection, at create on both ranks, and the voting rejection at ResetParameter"""
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(25, cat=True)
    half = len(X) // 2
    cases = [(o + " tree_learner=data num_machines=2", m) for o, m in ERRORS] + \
            [("interaction_constraints=[0,1] tree_learner=voting top_k=2 num_machines=2", "does not support interaction_constraints")]

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
                    b.reset_parameter("interaction_constraints=[0,1]")
                msgs.append(str(e.value))
                after = b.save_model_to_string()
                b.update_one_iter()
                return msgs, before == after, b.save_model_to_string()
            finally:
                b.free()
        finally:
            ds.free()

    res, errs = tc.on_ranks(2, 29860, body)
    assert not errs, errs
    for msgs, unchanged, model in res:
        for (_, want), got in zip(cases + [(None, "does not support interaction_constraints")], msgs):
            assert want in got, (want, got)
        assert unchanged
        assert "[interaction_constraints: ]" in model
    assert tc.trees(res[0][2]) == tc.trees(res[1][2])


def test_reset_cannot_leave_the_voting_learner(built):
    """the learner is chosen at create, so a reset that also asks for tree_learner=data still meets the voting checks.  Nothing trains
    after the resets: each must fail and leave the booster as it was."""
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(26, cat=True)
    half = len(X) // 2
    resets = [("tree_learner=data interaction_constraints=[0,1]", "does not support interaction_constraints"),
              ("tree_learner=data_parallel extra_trees=true", "does not support extra_trees"),
              ("tree_learner=data monotone_constraints=1,0,0,0,0", "does not support monotone_constraints")]

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ds = capi.Dataset.from_mat(X[sl], tc.ds_params(cats, 255)).set_field("label", np.asarray(-g[sl], np.float32))
        try:
            b = capi.Booster(ds, tc.params(8, "tree_learner=voting top_k=2 num_machines=2", cats))
            try:
                b.update_one_iter()
                before = b.save_model_to_string()
                out = []
                for opts, _ in resets:
                    with pytest.raises(Exception) as e:
                        b.reset_parameter(opts)
                    out.append((str(e.value), b.save_model_to_string() == before))
                return out
            finally:
                b.free()
        finally:
            ds.free()

    res, errs = tc.on_ranks(2, 29880, body)
    assert not errs, errs
    for out in res:
        for (_, want), (got, unchanged) in zip(resets, out):
            assert want in got and unchanged, (want, got, unchanged)


def test_model_text(built):
    X, g, h, cats = tc.data(8)
    dsp = tc.ds_params(cats, 255)
    model = tc.run(X, g, h, tc.params(8, "interaction_constraints=[0,2],[1],[]", cats), 2, dsp)
    assert "[interaction_constraints: [0,2],[1],[]]" in model
    assert "interaction_constraints" not in model.split("Tree=")[0]
    plain = tc.run(X, g, h, tc.params(8, "", cats), 2, dsp)
    assert "[interaction_constraints: ]" in plain


def test_estimator(built):
    """LightGBMRegressor(interactionConstraints=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    X, z = tc.monotone_data(5000, 10)
    X = np.nan_to_num(X)
    df = Frame({"features": X, "label": z})
    est = LightGBMRegressor(interactionConstraints=CONS, numIterations=5, numTasks=1)
    model = est.fit(df).getNativeModel()
    params = est.getTrainParams(1, df).to_string()
    assert params.endswith("interaction_constraints=[0,1],[1,2,3],[4] ")
    assert "interaction" not in LightGBMRegressor(numIterations=5).getTrainParams(1, df).to_string()
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
    assert tc.paths_inside(model, CONS) == 0
