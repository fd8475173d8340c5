"""Forced splits (forcedsplits_filename) on the GPU: every tree against the NumPy restatement (forced_splits_ref.grow_tree) on custom grid
gradients, the plan at the top of every tree on the objectives' own gradients, and the parameter's checks, aliases and equalities."""
import json
import os

import numpy as np
import pytest

import bynode_ref as B
import extra_trees_ref as X3
import forced_splits_ref as FS
import quant_ref as Q
import split_scan_ref as ref
import tree_check as C

pytestmark = pytest.mark.gpu


def _node(f, t, left=None, right=None):
    d = {"feature": f, "threshold": t}
    if left is not None:
        d["left"] = left
    if right is not None:
        d["right"] = right
    return d


def _write(tmp_path, plan, name="plan.json"):
    path = os.path.join(str(tmp_path), name)
    with open(path, "w") as fh:
        fh.write(plan if isinstance(plan, str) else json.dumps(plan))
    return path


def check_forced(tmp_path, X, g, h, cats, plan, num_leaves=8, iters=2, max_bin=255, extra="", fraction=1.0, max_depth=-1, cons=None,
                 extra_seed=None, phase_end=None, bynode=None, smooth=0.0, quant=None):
    """`iters` trees on the same custom (g, h) with the plan, each against forced_splits_ref.grow_tree.  bynode: feature_fraction_bynode;
    smooth: path_smooth; quant = (B, seed): use_quantized_grad with B levels and stochastic rounding, each tree against the restatement
    on quant_ref's levels times their scales (the caller keeps the scales powers of two, so the sums are exact)"""
    from mmlspark_b200.modeltext import parse_model
    path = _write(tmp_path, plan)
    opts = extra + " forcedsplits_filename=" + path
    if fraction < 1.0:
        opts += " feature_fraction=%r" % fraction
    if max_depth > 0:
        opts += " max_depth=%d" % max_depth
    if cons is not None:
        opts += " " + C.ic(cons)
    if extra_seed is not None:
        opts += " extra_trees=true extra_seed=%d" % extra_seed
    if bynode is not None:
        opts += " feature_fraction_bynode=%r" % bynode
    if smooth:
        opts += " path_smooth=%r" % smooth
    if quant is not None:
        opts += " use_quantized_grad=true num_grad_quant_bins=%d data_random_seed=%d" % quant
    model = C.run(X, g, h, C.params(num_leaves, opts, cats, max_bin), iters, C.ds_params(cats, max_bin))
    feats, bins, ub, b2c = C.dataset(X, cats, max_bin)
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(**dict({"min_data_in_leaf": 20}, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS}))
    nodes = FS.with_bins(FS.flatten(plan), feats, ub, b2c)
    used = X3.feature_fraction_sets(len(feats), fraction, 2, iters)
    streams = X3.Streams(feats, extra_seed) if extra_seed is not None else None
    sampler = B.ColSampler(feats, fraction, bynode) if bynode is not None else None
    trees = parse_model(model)["trees"]
    assert len(trees) == iters
    Ts = []
    for k in range(iters):
        gk, hk = g, h
        if quant is not None:
            qg, qh, s_g, s_h = Q.quantize(g.astype(np.float32), h.astype(np.float32), quant[0], True, quant[1], k)
            gk, hk = qg * s_g, qh * s_h
        T = FS.grow_tree(bins, gk, hk, feats, p, num_leaves, nodes, used=None if sampler is not None else {feats[i].real_index for i in used[k]},
                         streams=streams, constraints=cons, max_depth=max_depth, sampler=sampler, smooth=smooth)
        why = FS.undecided(T)
        assert not why, "tree %d does not discriminate:\n%s" % (k, "\n".join(why[:10]))
        if phase_end is not None:
            assert T["phase_end"] == phase_end, (T["phase_end"], T["forced"])
        C.compare_tree(trees[k], T, ub, b2c)
        Ts.append(T)
    return model, Ts


PLAN1 = _node(0, 30.5)
PLAN2 = _node(2, 4.0, _node(0, 20.5), _node(0, 40.5))
PLAN3 = _node(2, 4.0, _node(0, 20.5, _node(1, 0.25)), _node(0, 40.5, None, _node(1, -0.5)))


@pytest.mark.parametrize("plan", [PLAN1, PLAN2, PLAN3], ids=["depth1", "depth2", "depth3"])
def test_numerical_plans(tmp_path, plan):
    X, g, h, cats = C.data(1)
    _, Ts = check_forced(tmp_path, X, g, h, cats, plan, num_leaves=12)
    assert Ts[0]["phase_end"] == "plan" and Ts[0]["forced"] == list(range(len(FS.flatten(plan))))


def test_nan_feature(tmp_path):
    X, g, h, cats = C.data(2)
    check_forced(tmp_path, X, g, h, cats, _node(1, 0.1, _node(1, -1.0)), phase_end="plan")


def test_categorical_one_hot_and_many_vs_many(tmp_path):
    X, g, h, cats = C.data(3, cat=True)
    check_forced(tmp_path, X, g, h, cats, _node(3, 1, _node(4, 7), _node(4, 21)), num_leaves=10, phase_end="plan")


def test_unseen_category_ends_the_phase(tmp_path):
    X, g, h, cats = C.data(4, cat=True)
    check_forced(tmp_path, X, g, h, cats, _node(2, 4.0, _node(4, 97)), phase_end="invalid")


def test_bundle_member(tmp_path):
    rng = np.random.default_rng(5)
    n = 6000
    X, g, h, _ = C.data(5, n=n)
    sparse = np.zeros((n, 2))
    hot = rng.random(n) < 0.2
    sparse[hot, 0] = rng.integers(1, 20, hot.sum())      # never nonzero together: bundled
    sparse[~hot & (rng.random(n) < 0.2), 1] = 3.0
    X = np.hstack([X, sparse])
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, C.ds_params([], 255))
    try:
        _, col = ds.bundles()
    finally:
        ds.free()
    assert col[3] == col[4] >= 0      # the two sparse features share one storage column
    check_forced(tmp_path, X, g, h, [], _node(3, 8.5, _node(4, 1.5), _node(0, 30.5)), num_leaves=10)
    models = []
    for bundle in ("true", "false"):
        path = _write(tmp_path, _node(3, 8.5, _node(4, 1.5), _node(0, 30.5)), "b.json")
        models.append(C.run(X, g, h, C.params(10, "forcedsplits_filename=%s enable_bundle=%s" % (path, bundle)), 3,
                            C.DS + " max_bin=255 enable_bundle=" + bundle))
    assert C.trees(models[0]) == C.trees(models[1])


def test_wide_features(tmp_path):
    X, g, h, cats = C.data(6, wide=True)
    check_forced(tmp_path, X, g, h, cats, _node(3, 250.5, _node(5, 30), _node(4, 0.0)), max_bin=511, phase_end="plan")


def test_invalid_node_mid_plan(tmp_path):
    X, g, h, cats = C.data(7)
    # node 2 puts every row of its leaf on one side: no gain over the leaf, so the phase ends there and that round picks normally
    check_forced(tmp_path, X, g, h, cats, _node(2, 4.0, _node(0, 20.5), _node(0, 1000.0, _node(1, 0.0))),
                 extra="min_gain_to_split=0.001", phase_end="invalid")


def test_plan_deeper_than_max_depth(tmp_path):
    X, g, h, cats = C.data(8)
    check_forced(tmp_path, X, g, h, cats, PLAN3, max_depth=2, phase_end="unscanned")


def test_small_leaves(tmp_path):
    X, g, h, cats = C.data(9, n=400)
    # min_data_in_leaf=150: the children of the first split hold fewer than 2 * 150 rows, so they are never scanned
    check_forced(tmp_path, X, g, h, cats, _node(0, 30.5, _node(2, 4.0)), extra="min_data_in_leaf=150", phase_end="unscanned")


def test_plan_larger_than_the_tree(tmp_path):
    X, g, h, cats = C.data(10)
    check_forced(tmp_path, X, g, h, cats, PLAN3, num_leaves=3, phase_end="full")


def test_feature_outside_the_feature_fraction_sample(tmp_path):
    X, g, h, cats = C.data(11)
    _, Ts = check_forced(tmp_path, X, g, h, cats, _node(0, 30.5, _node(1, 0.0), _node(2, 2.0)), fraction=0.5, iters=3)
    assert all(T["phase_end"] == "plan" for T in Ts)


def test_interaction_constraints_and_extra_trees(tmp_path):
    X, g, h, cats = C.data(12)
    check_forced(tmp_path, X, g, h, cats, _node(0, 30.5, _node(1, 0.0)), cons=[[0, 2], [1]], extra_seed=9, iters=3, phase_end="plan")


def test_l1_and_max_delta_step(tmp_path):
    X, g, h, cats = C.data(13)
    # with outputs clamped to 0.8 the plan's last node gains nothing over its leaf, so the phase ends there
    check_forced(tmp_path, X, g, h, cats, PLAN2, extra="lambda_l1=0.5 max_delta_step=0.8", phase_end="invalid")


@pytest.mark.parametrize("smooth", [0.5, 10.0])
def test_path_smooth(tmp_path, smooth):
    """the output-based scans: the forced node's gain, min_gain_shift and children's outputs smoothed toward the leaf's output"""
    X, g, h, cats = C.data(15, cat=True)
    check_forced(tmp_path, X, g, h, cats, _node(2, 4.0, _node(0, 20.5), _node(3, 1)), num_leaves=10, smooth=smooth, iters=3,
                 phase_end="plan")


def test_feature_fraction_bynode(tmp_path):
    """the forced features are split whether or not a leaf's node sample holds them; the samples' draws are those of a plain run"""
    X, g, h, cats = C.data(16)
    _, Ts = check_forced(tmp_path, X, g, h, cats, _node(0, 30.5, _node(1, 0.0), _node(2, 2.0)), bynode=0.4, iters=4)
    assert all(T["phase_end"] == "plan" for T in Ts)


def test_quantized_grad(tmp_path):
    """quantised training: the forced nodes are evaluated on the packed histograms' levels, with stochastic draws per tree"""
    X, g, h, cats = C.data(17)
    g = np.clip(g, -2, 2); g[0] = 2.0      # |g| and |h| peak at 2 and 4: with B = 16 the scales are 2 / 8 and 4 / 16
    h = h * 2; h[0] = 4.0
    check_forced(tmp_path, X, g, h, cats, PLAN2, num_leaves=10, quant=(16, 5), iters=3, phase_end="plan")


# ---------------------------------------------------------------- the objectives' own gradients
def _top_nodes(model, nodes):
    """every tree's first len(nodes) splits against the plan: feature and the node each split was applied to"""
    from mmlspark_b200.modeltext import parse_model
    for t in parse_model(model)["trees"]:
        sf = t["split_feature"].tolist()
        assert sf[:len(nodes)] == [n["feature"] for n in nodes], sf


@pytest.mark.parametrize("case", ["regression", "binary", "multiclass", "lambdarank", "goss", "dart", "rf", "bagging"])
def test_objectives_start_every_tree_with_the_plan(tmp_path, case):
    from mmlspark_b200 import capi
    opts, K, label, n = C.CASES[case]
    n = min(n, 20000)
    X, z = C.monotone_data(n, 3)
    plan = _node(2, 25.5, _node(0, 0.0), _node(3, 0.0))
    path = _write(tmp_path, plan)
    ds = capi.Dataset.from_mat(X, C.DS).set_field("label", label(z).astype(np.float32))
    if case == "lambdarank":
        ds.set_field("group", np.full(n // 20, 20, np.int32))
    b = capi.Booster(ds, opts + " verbosity=-1 num_leaves=15 forcedsplits_filename=" + path)
    try:
        for _ in range(4):
            b.update_one_iter()
        model = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    _top_nodes(model, FS.flatten(plan))
    assert model.count("Tree=") == 4 * K


# ---------------------------------------------------------------- the parameter
def _train(X, y, params, iters=3):
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, C.DS).set_field("label", y.astype(np.float32))
    b = capi.Booster(ds, "objective=regression verbosity=-1 num_leaves=8 " + params)
    try:
        for _ in range(iters):
            b.update_one_iter()
        return b.save_model_to_string(), b.predict_device(X)
    finally:
        b.free(); ds.free()


def test_empty_value_and_no_key_are_identical():
    X, z = C.monotone_data(5000, 4)
    assert _train(X, z, "")[0] == _train(X, z, "forcedsplits_filename=")[0]


@pytest.mark.parametrize("key", ["forcedsplits_filename", "fs", "forced_splits_filename", "forced_splits_file", "forced_splits"])
def test_aliases_and_params_block(tmp_path, key):
    X, z = C.monotone_data(5000, 4)
    path = _write(tmp_path, _node(2, 10.5))
    model, _ = _train(X, z, "%s=%s" % (key, path))
    assert "[forcedsplits_filename: %s]" % path in model
    _top_nodes(model, [{"feature": 2}])


def test_save_load_and_host_predictions(tmp_path):
    from mmlspark_b200 import capi
    X, z = C.monotone_data(5000, 5)
    path = _write(tmp_path, _node(2, 10.5, _node(0, 0.5)))
    model, pred = _train(X, z, "forcedsplits_filename=" + path)
    b = capi.Booster(model_str=model)
    try:
        assert b.save_model_to_string() == model
        np.testing.assert_allclose(b.predict_for_mat(X).ravel(), np.asarray(pred).ravel(), rtol=1e-12, atol=1e-12)
    finally:
        b.free()


BAD = [
    ("missing", None, "cannot read"),
    ("malformed", '{"feature": 0, "threshold": ', "unexpected end"),
    ("float feature", '{"feature": 0.5, "threshold": 1}', "integer"),
    ("string feature", '{"feature": "0", "threshold": 1}', "integer"),
    ("feature out of range", '{"feature": 99, "threshold": 1}', "outside"),
    ("negative feature", '{"feature": -1, "threshold": 1}', "outside"),
    ("threshold", '{"feature": 0, "threshold": "a"}', "number"),
    ("child threshold", '{"feature": 0, "threshold": 1, "left": {"feature": 1, "threshold": null}}', "number"),
    ("unused feature", '{"feature": 5, "threshold": 1}', "not used"),
]


@pytest.mark.parametrize("name,text,msg", BAD, ids=[b[0] for b in BAD])
def test_errors_at_create_and_reset(tmp_path, name, text, msg):
    from mmlspark_b200 import capi
    X, z = C.monotone_data(3000, 6)
    X = np.hstack([X, np.ones((len(X), 1))])      # feature 5 is trivial: the dataset does not use it
    path = os.path.join(str(tmp_path), "absent.json") if text is None else _write(tmp_path, text)
    ds = capi.Dataset.from_mat(X, C.DS).set_field("label", z.astype(np.float32))
    try:
        with pytest.raises(Exception, match=msg):
            capi.Booster(ds, "objective=regression verbosity=-1 forcedsplits_filename=" + path)
        b = capi.Booster(ds, "objective=regression verbosity=-1 num_leaves=8")
        try:
            b.update_one_iter()
            before = b.save_model_to_string()
            with pytest.raises(Exception, match=msg):
                b.reset_parameter("forcedsplits_filename=" + path)
            assert b.save_model_to_string() == before      # the params block too: the reset changed nothing
            b.update_one_iter()
        finally:
            b.free()
    finally:
        ds.free()


def test_monotone_constraints_are_rejected(tmp_path):
    from mmlspark_b200 import capi
    X, z = C.monotone_data(3000, 7)
    path = _write(tmp_path, _node(2, 10.5))
    ds = capi.Dataset.from_mat(X, C.DS).set_field("label", z.astype(np.float32))
    try:
        with pytest.raises(Exception, match="monotone_constraints"):
            capi.Booster(ds, "objective=regression verbosity=-1 monotone_constraints=1,0,0,0,0 forcedsplits_filename=" + path)
        b = capi.Booster(ds, "objective=regression verbosity=-1 forcedsplits_filename=" + path)
        try:
            with pytest.raises(Exception, match="monotone_constraints"):
                b.reset_parameter("monotone_constraints=1,0,0,0,0")
        finally:
            b.free()
    finally:
        ds.free()


def test_reset_sets_changes_and_clears_the_plan(tmp_path):
    X, g, h, cats = C.data(14)
    p1, p2 = _write(tmp_path, PLAN1, "a.json"), _write(tmp_path, PLAN2, "b.json")
    from mmlspark_b200.modeltext import parse_model
    feats, bins, ub, b2c = C.dataset(X, cats, 255)
    p = ref.Params(min_data_in_leaf=20)
    seq = [None, p1, p2, ""]      # tree k is grown after the k-th reset (none before tree 0)
    model = None
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, C.ds_params(cats, 255)).set_field("label", np.zeros(len(X), np.float32))
    b = capi.Booster(ds, C.params(8, "", cats))
    try:
        for k, path in enumerate(seq):
            if path is not None:
                b.reset_parameter("forcedsplits_filename=" + path)
            b.update_one_iter_custom(g.astype(np.float32), h.astype(np.float32))
        model = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    trees = parse_model(model)["trees"]
    for k, plan in enumerate([None, PLAN1, PLAN2, None]):
        nodes = FS.with_bins(FS.flatten(plan), feats, ub, b2c) if plan else []
        T = FS.grow_tree(bins, g, h, feats, p, 8, nodes)
        assert not FS.undecided(T)
        C.compare_tree(trees[k], T, ub, b2c)


def test_two_ranks_give_the_one_rank_model(tmp_path):
    X, z = C.monotone_data(20000, 8)
    path = _write(tmp_path, _node(2, 25.5, _node(0, 0.0)))
    params = "objective=regression verbosity=-1 num_leaves=15 tree_learner=data forcedsplits_filename=" + path
    one = C.boost(X, z, params, 3, C.DS)
    two = C.boost(X, z, params, 3, C.DS, rank_rows=[10000, 10000], port=46310)
    assert C.trees(one) == C.trees(two)


def test_ranks_given_different_plans_fail_together(tmp_path):
    from mmlspark_b200 import capi
    X, z = C.monotone_data(4000, 9)
    paths = [_write(tmp_path, _node(2, 25.5), "r0.json"), _write(tmp_path, _node(2, 10.5), "r1.json")]
    half = len(X) // 2

    def body(r):
        full = capi.Dataset.from_mat(X, C.DS)
        ds = capi.Dataset.from_mat(X[r * half:(r + 1) * half], C.DS, reference=full).set_field("label", z[r * half:(r + 1) * half].astype(np.float32))
        try:
            capi.Booster(ds, "objective=regression verbosity=-1 tree_learner=data forcedsplits_filename=" + paths[r])
        finally:
            ds.free(); full.free()

    _, errs = C.on_ranks(2, 46320, body)
    assert sorted(r for r, _ in errs) == [0, 1]
    assert all("different forced split plans" in str(e) for _, e in errs)


def test_estimator(tmp_path):
    """LightGBMRegressor(forcedSplitsFilename=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    X, z = C.monotone_data(5000, 11)
    X = np.nan_to_num(X)
    path = _write(tmp_path, _node(2, 25.5, _node(4, 0.0)))
    df = Frame({"features": X, "label": z})
    est = LightGBMRegressor(forcedSplitsFilename=path, numIterations=5, numTasks=1)
    model = est.fit(df).getNativeModel()
    params = est.getTrainParams(1, df).to_string()
    assert "forcedsplits_filename=%s " % path in params
    assert "forcedsplits_filename" not in LightGBMRegressor(numIterations=5, numTasks=1).getTrainParams(1, df).to_string()
    ds = capi.Dataset.from_mat(X, dataset_params(est.get("maxBin"), est.get("binSampleCount"), est.get("numThreads"), []))
    ds.set_field("label", z.astype(np.float32))
    b = capi.Booster(ds, params)
    try:
        for _ in range(5):
            b.update_one_iter()
        low = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    assert C.trees(model) == C.trees(low)
    _top_nodes(model, [{"feature": 2}, {"feature": 4}])
    assert "[forcedsplits_filename: %s]" % path in model


def test_errors_fire_on_every_rank(tmp_path):
    """with two rank-threads: a bad plan on both ranks, the voting rejection at create, and the voting rejection at ResetParameter, on
    both ranks, each reset leaving the booster unchanged"""
    from mmlspark_b200 import capi
    X, g, h, cats = C.data(50)
    X = np.hstack([X, np.ones((len(X), 1))])      # feature 3 is trivial
    half = len(X) // 2
    good = _write(tmp_path, _node(0, 30.5), "good.json")
    cases = [("forcedsplits_filename=" + os.path.join(str(tmp_path), "absent.json"), "cannot read"),
             ("forcedsplits_filename=" + _write(tmp_path, "{", "bad.json"), "expected a string key"),
             ("forcedsplits_filename=" + _write(tmp_path, _node(3, 1.0), "unused.json"), "not used"),
             ("forcedsplits_filename=" + good + " tree_learner=voting top_k=2", "tree_learner=voting does not support forcedsplits_filename")]

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ds = capi.Dataset.from_mat(X[sl], C.ds_params(cats, 255)).set_field("label", np.asarray(-g[sl], np.float32))
        try:
            msgs = []
            for opts, _ in cases:
                with pytest.raises(Exception) as e:
                    capi.Booster(ds, C.params(8, "tree_learner=data num_machines=2 " + opts, cats))
                msgs.append(str(e.value))
            b = capi.Booster(ds, C.params(8, "tree_learner=voting top_k=2 num_machines=2", cats))
            try:
                b.update_one_iter()
                before = b.save_model_to_string()
                with pytest.raises(Exception) as e:
                    b.reset_parameter("forcedsplits_filename=" + good)
                msgs.append(str(e.value))
                unchanged = b.save_model_to_string() == before
                b.update_one_iter()
                return msgs, unchanged, b.save_model_to_string()
            finally:
                b.free()
        finally:
            ds.free()

    res, errs = C.on_ranks(2, 46330, body)
    assert not errs, errs
    wants = [m for _, m in cases] + ["tree_learner=voting does not support forcedsplits_filename"]
    for msgs, unchanged, model in res:
        assert len(msgs) == len(wants)
        for want, got in zip(wants, msgs):
            assert want in got, (want, got)
        assert unchanged
        assert "[forcedsplits_filename: ]" in model
    assert C.trees(res[0][2]) == C.trees(res[1][2])


@pytest.mark.parametrize("bad", ["absent", "malformed"])
def test_one_rank_cannot_load_its_plan(tmp_path, bad):
    """rank 1 cannot read or parse its file while rank 0 loads a good plan: both fail at create (rank 0 from the all-reduce) and neither
    waits; the same at ResetParameter, which leaves both boosters as they were"""
    from mmlspark_b200 import capi
    X, z = C.monotone_data(4000, 10)
    good = _write(tmp_path, _node(2, 25.5), "good.json")
    broken = os.path.join(str(tmp_path), "absent.json") if bad == "absent" else _write(tmp_path, '{"feature": 2,', "bad.json")
    paths = [good, broken]
    half = len(X) // 2

    def body(r):
        full = capi.Dataset.from_mat(X, C.DS)
        ds = capi.Dataset.from_mat(X[r * half:(r + 1) * half], C.DS, reference=full).set_field("label", z[r * half:(r + 1) * half].astype(np.float32))
        try:
            msgs = []
            with pytest.raises(Exception) as e:
                capi.Booster(ds, "objective=regression verbosity=-1 tree_learner=data num_machines=2 forcedsplits_filename=" + paths[r])
            msgs.append(str(e.value))
            b = capi.Booster(ds, "objective=regression verbosity=-1 num_leaves=8 tree_learner=data num_machines=2")
            try:
                b.update_one_iter()
                before = b.save_model_to_string()
                with pytest.raises(Exception) as e:
                    b.reset_parameter("forcedsplits_filename=" + paths[r])
                msgs.append(str(e.value))
                unchanged = b.save_model_to_string() == before
                b.update_one_iter()
                return msgs, unchanged
            finally:
                b.free()
        finally:
            ds.free(); full.free()

    res, errs = C.on_ranks(2, 46340 + (bad == "malformed") * 10, body)
    assert not errs, errs
    for msgs in res[0][0]:
        assert "another rank could not load" in msgs
    for msgs in res[1][0]:
        assert "forcedsplits_filename=" + broken in msgs
    assert res[0][1] and res[1][1]
