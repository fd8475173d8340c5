"""Path smoothing (path_smooth): the output-based scans (k_scan, k_scan_wide with kMono) smoothing every gain and min_gain_shift toward
the leaf's output, the pick step's smoothed outputs and the leaves' parent outputs, tree by tree against the NumPy restatement in
path_smooth_ref.py (grown by its grow_tree) on grid gradients and at the bar tree_check.py describes, on the engine's own gradients, and the
parameter checks, params block and estimator."""
import numpy as np
import pytest

import bynode_ref as B
import extra_trees_ref as X3
import interaction_ref as I
import path_smooth_ref as PS
import split_scan_ref as ref
import tree_check as tc

pytestmark = pytest.mark.gpu

CAT = "min_data_per_group=20 cat_smooth=5"


def _check_run(X, g, h, cats, num_leaves, iters, max_bin=255, extra="", smooth=None, extra_seed=None, mono=None, penalty=0.0, cons=None,
               bynode=None, max_depth=-1, reset=None):
    """tree_check.check_run with `smooth` (path_smooth): `iters` iterations on the same custom (g, h), every tree against
    path_smooth_ref.grow_tree with the same options, carried from tree to tree; reset = (after tree k, parameter string) calls
    ResetParameter, whose path_smooth replaces `smooth`.  min_data_in_leaf may be among the extra parameters; the restatement takes
    it raised to 2 while smoothing is on."""
    from mmlspark_b200.modeltext import parse_model
    opts = extra
    if smooth is not None:
        opts += " path_smooth=%r" % smooth
    if extra_seed is not None:
        opts += " extra_trees=true extra_seed=%d" % extra_seed
    if mono is not None:
        opts += " %s monotone_penalty=%r" % (tc.mc(mono), penalty)
    if cons is not None:
        opts += " " + tc.ic(cons)
    if bynode is not None:
        opts += " feature_fraction_bynode=%r" % bynode
    if max_depth > 0:
        opts += " max_depth=%d" % max_depth
    model = tc.run(X, g, h, tc.params(num_leaves, opts, cats, max_bin), iters, tc.ds_params(cats, max_bin), reset)
    feats, bins, ub, b2c = tc.dataset(X, cats, max_bin)
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(**dict({"min_data_in_leaf": 20}, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS}))
    min_data = p.min_data_in_leaf
    trees = parse_model(model)["trees"]
    assert len(trees) == iters
    sampler = B.ColSampler(feats, 1.0, bynode) if bynode is not None else None
    streams = X3.Streams(feats, extra_seed) if extra_seed is not None else None
    Ts = []
    for k in range(iters):
        if reset is not None and k == reset[0] + 1:
            streams = X3.Streams(feats, extra_seed) if extra_seed is not None else None      # ResetParameter re-seeds them
            smooth = float(dict(tok.split("=", 1) for tok in reset[1].split())["path_smooth"])
        p.min_data_in_leaf = PS.min_data_in_leaf(smooth or 0.0, min_data)
        T = PS.grow_tree(bins, g, h, feats, p, num_leaves, smooth=smooth or 0.0, streams=streams, mono=mono, penalty=penalty,
                         constraints=cons, sampler=sampler, max_depth=max_depth)
        why = ref.undecided(T)
        assert not why, "tree %d does not discriminate:\n%s" % (k, "\n".join(why[:10]))
        Ts.append(T)
        tc.compare_tree(trees[k], T, ub, b2c)
        for path in I.leaf_paths(trees[k]) if cons is not None else ():
            assert any(set(path) <= set(c) for c in cons), (k, path)
    return model, Ts


# ---------------------------------------------------------------- tree by tree against the restatement
@pytest.mark.parametrize("smooth", [0.5, 10.0, 1e6])
def test_numerical_with_nan(built, smooth):
    X, g, h, cats = tc.data(31)
    model, Ts = _check_run(X, g, h, cats, 12, 3, smooth=smooth)
    assert tc.split_features(model) >= {0, 1}
    assert "[path_smooth: %g]" % smooth in model


def test_categoricals(built):
    X, g, h, cats = tc.data(32, cat=True)
    g = g - 2.0 * (X[:, 4] % 2 == 0) - 1.0 * (X[:, 3] == 1)      # strong categorical signals, still on the grid
    model, _ = _check_run(X, g, h, cats, 16, 3, smooth=5.0, extra=CAT)
    assert tc.split_features(model) >= {3, 4}, "the case must split on the one-hot and the many-vs-many feature"


def test_wide_features(built):
    """max_bin=511: k_scan_wide's numerical scan and a wide categorical feature, smoothed"""
    X, g, h, cats = tc.data(33, n=9000, wide=True)
    model, _ = _check_run(X, g, h, cats, 12, 2, max_bin=511, smooth=3.0, extra=CAT)
    assert tc.split_features(model) & {3, 5}


def test_l1_and_max_delta_step(built):
    X, g, h, cats = tc.data(34)
    _check_run(X, g, h, cats, 12, 2, smooth=2.0, extra="lambda_l1=0.5 lambda_l2=1.0 max_delta_step=0.8")


@pytest.mark.parametrize("penalty", [0.0, 1.5])
def test_with_monotone_constraints(built, penalty):
    X, g, h, cats = tc.data(35, cat=True)
    _check_run(X, g, h, cats, 12, 3, mono=[1, 1, 1, 0, 0], penalty=penalty, smooth=4.0, extra=CAT)


def test_with_extra_trees(built):
    X, g, h, cats = tc.data(36, cat=True)
    _check_run(X, g, h, cats, 12, 4, extra_seed=5, smooth=4.0, extra=CAT)


def test_with_interaction_constraints_bynode_and_max_depth(built):
    X, g, h, cats = tc.data(37, cat=True)
    _check_run(X, g, h, cats, 12, 3, cons=[[0, 1, 3], [1, 2, 4]], smooth=2.0, extra=CAT)
    _check_run(X, g, h, cats, 12, 3, bynode=0.6, smooth=2.0, extra=CAT)
    _check_run(X, g, h, cats, 12, 3, max_depth=3, smooth=2.0, extra=CAT)


def test_reset_parameter_sets_changes_and_clears(built):
    X, g, h, cats = tc.data(38)
    model, _ = _check_run(X, g, h, cats, 12, 3, reset=(0, "path_smooth=3"))
    assert "[path_smooth: 3]" in model
    model, _ = _check_run(X, g, h, cats, 12, 3, smooth=1.0, reset=(0, "path_smooth=20"))
    assert "[path_smooth: 20]" in model
    model, _ = _check_run(X, g, h, cats, 12, 3, smooth=1.0, reset=(1, "path_smooth=0"))
    assert "[path_smooth: 0]" in model


# ---------------------------------------------------------------- off is the unsmoothed engine, bit for bit
@pytest.mark.parametrize("off", ["path_smooth=0", "path_smooth=1e-16"])
def test_off_is_bit_identical(built, off):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(39, cat=True)
    dsp = tc.ds_params(cats, 255)
    y = -g
    models, scores = [], []
    for opts in ("", off):
        params = "objective=regression num_leaves=16 learning_rate=0.3 verbosity=-1 metric= %s %s %s" % (dsp, CAT, opts)
        ds = capi.Dataset.from_mat(X, dsp).set_field("label", y.astype(np.float32))
        b = capi.Booster(ds, params)
        try:
            for _ in range(4):
                b.update_one_iter()
            models.append(b.save_model_to_string())
            scores.append(b.predict_device(X, capi.PREDICT_RAW_SCORE))
        finally:
            b.free(); ds.free()
    assert tc.trees(models[0]) == tc.trees(models[1])
    assert np.array_equal(scores[0], scores[1])


# ---------------------------------------------------------------- boosting runs on the engine's own gradients
def _check_boosting(X, y, objective, K, iters, extra, cats=(), fraction=1.0, bag=None, group=None, rank_rows=None, port=None, smooth=2.0):
    """every tree of the run equals path_smooth_ref.grow_tree on the gradients it was grown from (quantised as K3 does), over its bagged rows;
    rf grows every tree from the gradients at the initial scores (RF::Init) and does not shrink it"""
    from mmlspark_b200.modeltext import parse_model
    lr, num_leaves = 0.3, 12
    dsp = tc.ds_params(cats, 255)
    params = ("objective=%s boost_from_average=false learning_rate=%g num_leaves=%d min_data_in_leaf=20 verbosity=-1 metric= "
              "path_smooth=%r %s %s" % (objective, lr, num_leaves, smooth, dsp, extra))
    if rank_rows:
        params += " tree_learner=data num_machines=%d" % len(rank_rows)
    model, grads, const_h = tc.boost(X, y, params, iters, dsp, group=group, rank_rows=rank_rows, port=port, grads=True)
    feats, bins, ub, b2c = tc.dataset(X, cats, 255)
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(min_data_in_leaf=20, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS})
    trees = parse_model(model)["trees"]
    assert len(trees) == iters * K
    used = X3.feature_fraction_sets(len(feats), fraction, 2, iters * K)
    bags = tc.bags(len(X), iters, bag[0], bag[1]) if bag else None
    rf = "boosting=rf" in extra
    for it in range(iters):
        for k in range(K):
            gi = 0 if rf else it
            g = grads[gi][0].reshape(K, -1)[k]
            h = grads[gi][1].reshape(K, -1)[k]
            gq, hq = tc.quantized(g), (np.ones(len(h)) if const_h else tc.quantized(h))
            rows = np.arange(len(g)) if bags is None else np.nonzero(bags[it])[0]
            T = PS.grow_tree(bins[rows], gq[rows], hq[rows], feats, p, num_leaves, smooth=smooth,
                                   used={feats[i].real_index for i in used[it * K + k]})
            why = ref.undecided(T)
            assert not why, "iteration %d class %d does not discriminate:\n%s" % (it, k, "\n".join(why[:10]))
            tc.compare_tree(trees[it * K + k], T, ub, b2c, None if rf else lr)
    return model


def test_boosting_regression(built):
    X, g, h, cats = tc.data(40)
    _check_boosting(X, -g, "regression", 1, 4, "")


def test_boosting_binary_categorical(built):
    X, g, h, cats = tc.data(41, cat=True)
    X[:, 1] = np.nan_to_num(X[:, 1])      # NaN is covered above; here an empty NaN bin would tie both passes
    z = -g + 3.0 * (X[:, 4] % 2 == 0) + 2.0 * (X[:, 3] == 1)
    _check_boosting(X, (z > np.median(z)).astype(np.float64), "binary", 1, 4, CAT, cats)


def test_boosting_multiclass(built):
    X, g, h, cats = tc.data(42, cat=True)
    X[:, 1] = np.nan_to_num(X[:, 1])      # NaN is covered above; here an empty NaN bin would tie both passes
    y = np.digitize(-g, np.quantile(-g, [1 / 3, 2 / 3])).astype(np.float64)
    _check_boosting(X, y, "multiclass", 3, 3, "num_class=3 " + CAT, cats)


def test_boosting_lambdarank(built):
    X, g, h, cats = tc.data(43)
    X[:, 1] = np.nan_to_num(X[:, 1])      # NaN is covered above; here an empty NaN bin would tie both passes
    y = np.digitize(-g, np.quantile(-g, [0.5, 0.8, 0.95])).astype(np.float64)
    _check_boosting(X, y, "lambdarank", 1, 3, "", group=[20] * (len(X) // 20))


def test_boosting_bagging(built):
    X, g, h, cats = tc.data(44, cat=True)
    _check_boosting(X, -g, "regression", 1, 4, "bagging_fraction=0.6 bagging_freq=1 bagging_seed=7 feature_fraction=0.7 " + CAT, cats,
                    fraction=0.7, bag=(0.6, 7))


def test_boosting_rf(built):
    X, g, h, cats = tc.data(45)
    _check_boosting(X, -g, "regression", 1, 3, "boosting=rf bagging_fraction=0.7 bagging_freq=1 bagging_seed=3 feature_fraction=0.8",
                    fraction=0.8, bag=(0.7, 3))


def test_boosting_two_ranks_on_one_device(built):
    """data-parallel regression (unit hessians: the reconstructed global counts are exact) on two unequal shards"""
    X, g, h, cats = tc.data(46, cat=True)
    _check_boosting(X, -g, "regression", 1, 3, CAT, cats, rank_rows=[3100, 2900], port=29860)


@pytest.mark.parametrize("case", ["goss", "dart", "l1"])
def test_boosting_modes_smooth_and_differ(built, case):
    """GOSS, DART and regression_l1 (renewed leaves): smoothing trains, changes the model, and 1e-16 leaves it as the key left out"""
    X, g, h, cats = tc.data(47)
    dsp = tc.ds_params(cats, 255)
    opts = {"goss": "objective=regression boosting=goss", "dart": "objective=regression boosting=dart drop_rate=0.3",
            "l1": "objective=regression_l1"}[case]
    base = "%s num_leaves=16 learning_rate=0.3 verbosity=-1 metric= %s" % (opts, dsp)
    plain = tc.boost(X, -g, base, 4, dsp)
    tiny = tc.boost(X, -g, base + " path_smooth=1e-16", 4, dsp)
    smooth = tc.boost(X, -g, base + " path_smooth=20", 4, dsp)
    assert tc.trees(plain) == tc.trees(tiny)
    assert tc.trees(plain) != tc.trees(smooth)


# ---------------------------------------------------------------- ranks, bundles
def _two_ranks_match_one(port, device_of=lambda r: 0):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(48, const_h=True)
    dsp = tc.ds_params(cats, 255)
    params = tc.params(10, "tree_learner=data num_machines=2 path_smooth=3", cats)
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

    res, errs = tc.on_ranks(2, port, body, device_of)
    assert not errs, errs
    assert tc.trees(res[0]) == tc.trees(res[1])
    single, _ = _check_run(X, g, h, cats, 10, 3, smooth=3.0)
    assert tc.trees(res[0]) == tc.trees(single)


def test_two_ranks_equal_one(built):
    _two_ranks_match_one(29820)


def test_two_ranks_nccl(built):
    import subprocess
    out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
    if len([l for l in out.splitlines() if l.startswith("GPU ")]) < 2:
        pytest.skip("needs 2 GPUs")
    _two_ranks_match_one(29840, device_of=lambda r: r)


def test_bundles_equal_unbundled(built):
    rng = np.random.default_rng(19)
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
        models.append(tc.run(X, g, h, tc.params(12, "path_smooth=5 enable_bundle=" + bundle), 4, dsp))
    assert tc.trees(models[0]) == tc.trees(models[1])
    assert tc.split_features(models[0]) & {0, 1, 3}


# ---------------------------------------------------------------- errors, params block, estimator
ERRORS = [("path_smooth=-1", "path_smooth should be >= 0"), ("path_smooth=nan", "path_smooth should be >= 0")]


@pytest.mark.parametrize("opts,msg", ERRORS)
def test_create_and_reset_errors(built, opts, msg):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(49)
    ds = capi.Dataset.from_mat(X, tc.ds_params(cats, 255)).set_field("label", np.asarray(-g, np.float32))
    try:
        with pytest.raises(Exception) as e:
            capi.Booster(ds, tc.params(8, opts, cats))
        assert msg in str(e.value), str(e.value)
        b = capi.Booster(ds, tc.params(8, "path_smooth=2", cats))
        try:
            b.update_one_iter()
            before = b.save_model_to_string()
            with pytest.raises(Exception) as e:
                b.reset_parameter(opts)
            assert msg in str(e.value), str(e.value)
            assert b.save_model_to_string() == before and "[path_smooth: 2]" in before
        finally:
            b.free()
    finally:
        ds.free()


def test_errors_fire_on_every_rank(built):
    """each create-time error and the voting rejection, at create on both ranks, and the voting rejection at ResetParameter"""
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(50, cat=True)
    half = len(X) // 2
    cases = [(o + " tree_learner=data num_machines=2", m) for o, m in ERRORS] + \
            [("path_smooth=1 tree_learner=voting top_k=2 num_machines=2", "does not support path_smooth")]

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ds = capi.Dataset.from_mat(X[sl], tc.ds_params(cats, 255)).set_field("label", np.asarray(-g[sl], np.float32))
        try:
            msgs = []
            for opts, _ in cases:
                with pytest.raises(Exception) as e:
                    capi.Booster(ds, tc.params(8, opts, cats))
                msgs.append(str(e.value))
            b = capi.Booster(ds, tc.params(8, "tree_learner=voting top_k=2 num_machines=2 path_smooth=1e-16", cats))
            try:
                b.update_one_iter()
                before = b.save_model_to_string()
                for bad in ("path_smooth=1", "path_smooth=-1"):
                    with pytest.raises(Exception) as e:
                        b.reset_parameter(bad)
                    msgs.append(str(e.value))
                after = b.save_model_to_string()
                b.update_one_iter()
                return msgs, before == after, b.save_model_to_string()
            finally:
                b.free()
        finally:
            ds.free()

    res, errs = tc.on_ranks(2, 29880, body)
    assert not errs, errs
    wants = [m for _, m in cases] + ["does not support path_smooth", "path_smooth should be >= 0"]
    for msgs, unchanged, model in res:
        assert len(msgs) == len(wants)
        for want, got in zip(wants, msgs):
            assert want in got, (want, got)
        assert unchanged
        assert "[path_smooth: 1e-16]" in model
    assert tc.trees(res[0][2]) == tc.trees(res[1][2])


def test_params_block_and_round_trip(built):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(51)
    dsp = tc.ds_params(cats, 255)
    model = tc.run(X, g, h, tc.params(8, "path_smooth=2.5", cats), 2, dsp)
    assert "[path_smooth: 2.5]" in model and "[min_data_in_leaf: 20]" in model
    loaded = capi.Booster(model_str=model)
    try:
        assert loaded.save_model_to_string() == model
    finally:
        loaded.free()
    plain = tc.run(X, g, h, tc.params(8, "", cats), 2, dsp)
    assert "[path_smooth: 0]" in plain
    # CheckParamConflict: min_data_in_leaf is raised to 2 while smoothing is on, and the params block shows it
    raised = tc.run(X, g, h, tc.params(8, "path_smooth=1 min_data_in_leaf=1", cats), 1, dsp)
    assert "[min_data_in_leaf: 2]" in raised
    tiny = tc.run(X, g, h, tc.params(8, "path_smooth=1e-16 min_data_in_leaf=1", cats), 1, dsp)
    assert "[min_data_in_leaf: 1]" in tiny and "[path_smooth: 1e-16]" in tiny


def test_min_data_in_leaf_rule_trees(built):
    """min_data_in_leaf=1 with smoothing grows the restatement's trees at min_data_in_leaf=2"""
    X, g, h, cats = tc.data(52, n=400)
    X[:, 1] = np.nan_to_num(X[:, 1])      # with so few rows an empty NaN bin would tie both passes
    _check_run(X, g, h, cats, 8, 2, smooth=1.0, extra="min_data_in_leaf=1")


def test_estimator(built):
    """LightGBMRegressor(pathSmooth=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    X, z = tc.monotone_data(5000, 11)
    X = np.nan_to_num(X)
    df = Frame({"features": X, "label": z})
    est = LightGBMRegressor(pathSmooth=5.0, numIterations=5, numTasks=1)
    model = est.fit(df).getNativeModel()
    params = est.getTrainParams(1, df).to_string()
    assert params.endswith("path_smooth=5.0 ")
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
    assert "[path_smooth: 5]" in model
