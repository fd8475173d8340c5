"""Monotone constraints (monotone_constraints, monotone_penalty, basic method): the scans' kMono instantiations (k_scan, k_scan_wide), the
pick step's clamped outputs and the round controller's leaf bounds, tree by tree against the NumPy restatement in monotone_ref.py, and
the trained models' monotonicity on the engine's own gradients.

As in test_gpu_extra_trees.py, gradients and hessians lie on a 2^-10 grid with few enough rows that K4's fixed-point histograms equal
NumPy's fp64 ones bit for bit, so only the scans and the pick are under test.  Bar: identical structure, leaf values within 4 fp64 ulps,
split gains as printed, and every tree decided on the reference side (split_scan_ref.undecided)."""
import numpy as np
import pytest

import monotone_ref as M
import split_scan_ref as ref
import extra_trees_ref as X3
import test_gpu_extra_trees as ET

pytestmark = pytest.mark.gpu


def _mc(mono):
    return "monotone_constraints=" + ",".join(str(m) for m in mono)


def _check_run(X, g, h, cats, num_leaves, iters, mono, max_bin=255, extra="", penalty=0.0, extra_seed=None, reset=None):
    """`iters` trees on the same custom (g, h) against monotone_ref.grow_tree; reset = (after tree k, new constraint list) changes the
    constraints through ResetParameter"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import parse_model
    dsp = ET._ds_params(cats, max_bin)
    opts = "%s monotone_penalty=%r %s" % (_mc(mono), penalty, extra)
    if extra_seed is not None:
        opts += " extra_trees=true extra_seed=%d" % extra_seed
    model = ET._run(X, g, h, ET._params(num_leaves, opts, cats, max_bin), iters, dsp, None if reset is None else (reset[0], _mc(reset[1])))
    ds = capi.Dataset.from_mat(X, dsp).set_field("label", np.zeros(len(X), np.float32))
    try:
        feats = ET._features(ds, X.shape[1], cats)
        bins = ds.get_bins16()
        ub = {f.real_index: ds.upper_bounds(f.real_index) for f in feats}
        b2c = {f.real_index: ds.bin_to_cat(f.real_index) for f in feats if f.is_cat}
    finally:
        ds.free()
    kv = dict(tok.split("=", 1) for tok in extra.split())
    p = ref.Params(min_data_in_leaf=20, **{k: v for k, v in kv.items() if k in ref.Params.DEFAULTS})
    trees = parse_model(model)["trees"]
    assert len(trees) == iters
    streams = X3.Streams(feats, extra_seed) if extra_seed is not None else None
    for k in range(iters):
        m = mono if reset is None or k <= reset[0] else reset[1]
        if reset is not None and k == reset[0] + 1 and streams is not None:
            streams = X3.Streams(feats, extra_seed)
        T = M.grow_tree(bins, g, h, feats, p, num_leaves, m, penalty, extra_seed is not None, extra_seed or 6, streams)
        why = ref.undecided(T)
        assert not why, "tree %d does not discriminate:\n%s" % (k, "\n".join(why[:10]))
        ET._compare(trees[k], T, ub, b2c)
    return model


# ---------------------------------------------------------------- tree by tree against the restatement
def test_numerical_with_nan(built):
    X, g, h, cats = ET._data(1)
    X[:, 2] = -X[:, 2]      # the target falls with this feature: a -1 constraint still lets it split
    model = _check_run(X, g, h, cats, 12, 3, [1, 1, -1])
    assert ET._split_features(model) >= {1, 2}


def test_l1_and_max_delta_step(built):
    X, g, h, cats = ET._data(11)
    _check_run(X, g, h, cats, 12, 2, [-1, 1, 1], extra="lambda_l1=0.5 lambda_l2=1.0 max_delta_step=0.8")


def test_categoricals_in_constrained_leaves(built):
    X, g, h, cats = ET._data(2, cat=True)
    model = _check_run(X, g, h, cats, 16, 3, [1, -1, 1, 0, 0], extra="min_data_per_group=20 cat_smooth=5")
    assert ET._split_features(model) >= {3, 4}, "the case must split on the one-hot and the many-vs-many feature"


def test_wide_features(built):
    """max_bin=511: k_scan_wide's numerical scan under a constraint and a wide categorical feature in constrained leaves"""
    X, g, h, cats = ET._data(4, n=9000, wide=True)
    model = _check_run(X, g, h, cats, 12, 2, [1, -1, 0, 1, 0, 0], max_bin=511, extra="min_data_per_group=20 cat_smooth=5")
    assert 3 in ET._split_features(model)


@pytest.mark.parametrize("penalty", [0.5, 2.5])
def test_penalty(built, penalty):
    X, g, h, cats = ET._data(12)
    _check_run(X, g, h, cats, 12, 2, [1, -1, 1], penalty=penalty)


def test_extra_trees(built):
    X, g, h, cats = ET._data(13, cat=True)
    _check_run(X, g, h, cats, 12, 4, [1, -1, 0, 0, 0], extra="min_data_per_group=20 cat_smooth=5", extra_seed=9)


def test_all_zero_list(built):
    """an all-zero list runs the constrained scans: the restatement's USE_MC scans, gains from the outputs"""
    X, g, h, cats = ET._data(14, cat=True)
    _check_run(X, g, h, cats, 12, 2, [0, 0, 0, 0, 0], extra="min_data_per_group=20 cat_smooth=5")


def test_reset_parameter_changes_the_constraints(built):
    X, g, h, cats = ET._data(15)
    model = _check_run(X, g, h, cats, 12, 4, [1, 0, 0], reset=(1, [-1, -1, 1]))
    assert "[monotone_constraints: -1,-1,1]" in model


# ---------------------------------------------------------------- monotone predictions on the engine's own gradients
def _sweep_violations(predict, X, mono, K, rows=200, seed=0):
    """for `rows` base rows and every constrained feature, the raw scores over the feature's sorted distinct non-NaN values; returns the
    number of (row, feature, class) sweeps that break the direction, with no tolerance"""
    rng = np.random.default_rng(seed)
    base = X[rng.choice(len(X), rows, replace=False)]
    bad = 0
    for f, m in enumerate(mono):
        if m == 0:
            continue
        vals = np.unique(X[:, f][~np.isnan(X[:, f])])
        grid = np.repeat(base, len(vals), axis=0)
        grid[:, f] = np.tile(vals, rows)
        raw = np.asarray(predict(grid), np.float64).reshape(rows, len(vals), K)
        d = np.diff(raw, axis=1) * m
        bad += int((d < 0).any(axis=1).sum())
    return bad


def _boosted(X, y, params, iters, dsp, group=None, rank_rows=None, port=None):
    """trains on the engine's own gradients; returns the model text (every rank's, when data-parallel, must be equal)"""
    from mmlspark_b200 import capi
    rank_rows = rank_rows or [len(X)]
    offs = np.concatenate([[0], np.cumsum(rank_rows)])

    def body(r):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        full = capi.Dataset.from_mat(X, dsp)
        ds = capi.Dataset.from_mat(X[sl], dsp, reference=full).set_field("label", np.asarray(y[sl], np.float32))
        if group is not None:
            ds.set_field("group", np.asarray(group, np.int32))
        b = capi.Booster(ds, params)
        try:
            for _ in range(iters):
                b.update_one_iter()
            return b.save_model_to_string()
        finally:
            b.free(); ds.free(); full.free()

    if len(rank_rows) == 1:
        return body(0)
    res, errs = ET._on_ranks(len(rank_rows), port, body)
    assert not errs, errs
    assert all(ET._trees(r) == ET._trees(res[0]) for r in res)
    return res[0]


def _monotone_data(n, seed):
    rng = np.random.default_rng(seed)
    # a few hundred distinct values per constrained feature, so that a sweep over all of them stays small
    X = np.stack([rng.integers(-150, 150, n) / 50.0, rng.integers(-100, 100, n) / 50.0, rng.integers(0, 50, n).astype(np.float64),
                  rng.standard_normal(n), rng.standard_normal(n)], axis=1)
    X[rng.random(n) < 0.05, 0] = np.nan
    # against the constraints in places, so an unconstrained model breaks them
    z = np.sin(2 * np.nan_to_num(X[:, 0])) + 0.8 * np.nan_to_num(X[:, 0]) - np.cos(2 * X[:, 1]) - 0.6 * X[:, 1] \
        + 0.03 * X[:, 2] + 0.3 * np.sin(X[:, 2]) + X[:, 3] * X[:, 4] + 0.3 * rng.standard_normal(n)
    return X, z


MONO = [1, -1, 1, 0, 0]

CASES = {
    "regression": ("objective=regression", 1, lambda z: z, 50000),
    "binary": ("objective=binary", 1, lambda z: (z > np.median(z)).astype(float), 50000),
    "multiclass": ("objective=multiclass num_class=3", 3, lambda z: np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])).astype(float), 30000),
    "lambdarank": ("objective=lambdarank", 1, lambda z: np.digitize(z, np.quantile(z, [0.5, 0.8, 0.95])).astype(float), 20000),
    "goss": ("objective=regression boosting=goss", 1, lambda z: z, 50000),
    "dart": ("objective=regression boosting=dart drop_rate=0.3", 1, lambda z: z, 30000),
    "rf": ("objective=regression boosting=rf bagging_fraction=0.7 bagging_freq=1 feature_fraction=0.8", 1, lambda z: z, 50000),
    "bagging": ("objective=regression bagging_fraction=0.6 bagging_freq=1 feature_fraction=0.8", 1, lambda z: z, 200000),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_predictions_are_monotone(built, case):
    from mmlspark_b200 import capi
    obj, K, label, n = CASES[case]
    X, z = _monotone_data(n, 30 + len(case))
    y = label(z)
    group = [20] * (n // 20) if case == "lambdarank" else None
    dsp = ET.DS + " max_bin=255"
    base = "%s num_leaves=31 learning_rate=0.3 min_data_in_leaf=20 verbosity=-1 metric= %s" % (obj, dsp)
    for mono, want_monotone in ((MONO, True), (None, False)):
        params = base + (" " + _mc(mono) + " monotone_penalty=0.5" if mono else "")
        model = _boosted(X, y, params, 8, dsp, group)
        b = capi.Booster(model_str=model)
        try:
            dev = _sweep_violations(lambda A: b.predict_device(A, capi.PREDICT_RAW_SCORE), X, MONO, K)
            host = _sweep_violations(lambda A: b.predict_for_mat(A, capi.PREDICT_RAW_SCORE), X, MONO, K)
        finally:
            b.free()
        if want_monotone:
            assert dev == 0 and host == 0, (dev, host)
        else:
            assert dev > 0, "the unconstrained model must break the constraints, or the check would not bite"


def test_predictions_are_monotone_two_ranks_on_one_device(built):
    from mmlspark_b200 import capi
    X, z = _monotone_data(40000, 50)
    dsp = ET.DS + " max_bin=255"
    params = "objective=regression num_leaves=31 learning_rate=0.3 verbosity=-1 metric= tree_learner=data num_machines=2 %s %s" % (_mc(MONO), dsp)
    model = _boosted(X, z, params, 8, dsp, rank_rows=[21000, 19000], port=29700)
    b = capi.Booster(model_str=model)
    try:
        assert _sweep_violations(lambda A: b.predict_device(A, capi.PREDICT_RAW_SCORE), X, MONO, 1) == 0
    finally:
        b.free()


def _two_ranks_match_one(port, device_of=lambda r: 0):
    from mmlspark_b200 import capi  # noqa: F401
    X, g, h, cats = ET._data(6, const_h=True)
    dsp = ET._ds_params(cats, 255)
    params = ET._params(10, "tree_learner=data num_machines=2 monotone_penalty=0.5 " + _mc([1, -1, 1]), cats)
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

    res, errs = ET._on_ranks(2, port, body, device_of)
    assert not errs, errs
    assert ET._trees(res[0]) == ET._trees(res[1])
    single = _check_run(X, g, h, cats, 10, 3, [1, -1, 1], penalty=0.5)
    assert ET._trees(res[0]) == ET._trees(single)


def test_two_ranks_equal_one(built):
    _two_ranks_match_one(29720)


def test_two_ranks_nccl(built):
    import subprocess
    out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
    if len([l for l in out.splitlines() if l.startswith("GPU ")]) < 2:
        pytest.skip("needs 2 GPUs")
    _two_ranks_match_one(29740, device_of=lambda r: r)


# ---------------------------------------------------------------- bundles, errors, model text, estimator
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
    g = np.round((-(X[:, 0] * 0.2 + X[:, 3] * 0.1 - X[:, 1] * 0.15 + X[:, 6]) + 0.2 * rng.standard_normal(n)) / ET.GRID) * ET.GRID
    h = ET._grid(rng, 0.5, 1.5, n)
    mono = [1, -1, 0, 1, 0, 0, 1, -1]
    models = []
    for bundle in ("true", "false"):
        dsp = ET.DS + " max_bin=255 enable_bundle=" + bundle
        models.append(ET._run(X, g, h, ET._params(12, _mc(mono) + " enable_bundle=" + bundle), 4, dsp))
    assert ET._trees(models[0]) == ET._trees(models[1])
    assert ET._split_features(models[0]) & {0, 1, 3}


ERRORS = [
    ("monotone_constraints=1,-1", "has 2 entries, but the dataset has 5 features"),
    ("monotone_constraints=1,2,0,0,0", "should be -1, 0 or 1"),
    ("monotone_constraints=0,0,0,1,0", "is categorical"),
    ("monotone_constraints=1,0,0,0,0 monotone_penalty=-1", "monotone_penalty should be >= 0"),
    ("mc=1,0,0,0,0 monotone_constraints_method=intermediate", "monotone_constraints_method=intermediate is not supported"),
    ("monotone_constraint=1,0,0,0,0 mc_method=advanced", "monotone_constraints_method=advanced is not supported"),
]


@pytest.mark.parametrize("opts,msg", ERRORS)
def test_create_errors(built, opts, msg):
    from mmlspark_b200 import capi
    X, g, h, cats = ET._data(7, cat=True)
    ds = capi.Dataset.from_mat(X, ET._ds_params(cats, 255)).set_field("label", np.asarray(-g, np.float32))
    try:
        with pytest.raises(Exception) as e:
            capi.Booster(ds, ET._params(8, opts, cats))
        assert msg in str(e.value), str(e.value)
    finally:
        ds.free()


def test_errors_fire_on_every_rank(built):
    """each create-time error and the voting rejection, at create on both ranks, and the voting rejection at ResetParameter"""
    from mmlspark_b200 import capi
    X, g, h, cats = ET._data(25, cat=True)
    half = len(X) // 2
    cases = [(o + " tree_learner=data num_machines=2", m) for o, m in ERRORS] + \
            [("monotone_constraints=1,0,0,0,0 tree_learner=voting top_k=2 num_machines=2", "does not support monotone_constraints")]

    def body(r):
        sl = slice(r * half, (r + 1) * half)
        ds = capi.Dataset.from_mat(X[sl], ET._ds_params(cats, 255)).set_field("label", np.asarray(-g[sl], np.float32))
        try:
            msgs = []
            for opts, _ in cases:
                with pytest.raises(Exception) as e:
                    capi.Booster(ds, ET._params(8, opts, cats))
                msgs.append(str(e.value))
            b = capi.Booster(ds, ET._params(8, "tree_learner=voting top_k=2 num_machines=2", cats))
            try:
                b.update_one_iter()
                before = b.save_model_to_string()
                with pytest.raises(Exception) as e:
                    b.reset_parameter("monotone_constraints=1,0,0,0,0")
                msgs.append(str(e.value))
                after = b.save_model_to_string()
                b.update_one_iter()
                return msgs, before == after, b.save_model_to_string()
            finally:
                b.free()
        finally:
            ds.free()

    res, errs = ET._on_ranks(2, 29760, body)
    assert not errs, errs
    for msgs, unchanged, model in res:
        for (_, want), got in zip(cases + [(None, "does not support monotone_constraints")], msgs):
            assert want in got, (want, got)
        assert unchanged
        assert "[monotone_constraints: ]" in model and "monotone_constraints=" not in model.split("Tree=")[0]
    assert ET._trees(res[0][2]) == ET._trees(res[1][2])


def test_model_text_round_trips(built):
    from mmlspark_b200 import capi
    X, g, h, cats = ET._data(8)
    dsp = ET._ds_params(cats, 255)
    model = ET._run(X, g, h, ET._params(8, "mc=1,-1,0 monotone_constraints_method=basic ms_penalty=1.5", cats), 2, dsp)
    head = model.split("Tree=")[0]
    lines = head.splitlines()
    i = [k for k, l in enumerate(lines) if l.startswith("monotone_constraints=")]
    assert len(i) == 1 and lines[i[0]] == "monotone_constraints=1 -1 0"
    assert lines[i[0] - 1].startswith("feature_names=") and lines[i[0] + 1].startswith("feature_infos=")
    assert "[monotone_constraints: 1,-1,0]" in model and "[monotone_constraints_method: basic]" in model and "[monotone_penalty: 1.5]" in model
    loaded = capi.Booster(model_str=model)
    try:
        assert loaded.save_model_to_string() == model
    finally:
        loaded.free()
    plain = ET._run(X, g, h, ET._params(8, "", cats), 2, dsp)
    assert "monotone_constraints=" not in plain.split("Tree=")[0]
    assert "[monotone_constraints: ]" in plain and "[monotone_penalty: 0]" in plain


def test_estimator(built):
    """LightGBMRegressor(monotoneConstraints=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    X, z = _monotone_data(5000, 10)
    X = np.nan_to_num(X)
    df = Frame({"features": X, "label": z})
    est = LightGBMRegressor(monotoneConstraints=MONO, monotonePenalty=0.5, numIterations=5, numTasks=1)
    model = est.fit(df).getNativeModel()
    params = est.getTrainParams(1, df).to_string()
    assert params.endswith("monotone_constraints=1,-1,1,0,0 monotone_constraints_method=basic monotone_penalty=0.5 ")
    assert "monotone" not in LightGBMRegressor(numIterations=5).getTrainParams(1, df).to_string()
    ds = capi.Dataset.from_mat(X, dataset_params(est.get("maxBin"), est.get("binSampleCount"), est.get("numThreads"), []))
    ds.set_field("label", z.astype(np.float32))
    b = capi.Booster(ds, params)
    try:
        for _ in range(5):
            b.update_one_iter()
        low = b.save_model_to_string()
    finally:
        b.free(); ds.free()
    assert ET._trees(model) == ET._trees(low)
    assert "monotone_constraints=1 -1 1 0 0" in model
