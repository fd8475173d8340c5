"""Monotone constraints (monotone_constraints, monotone_penalty, basic method): the scans' kMono instantiations (k_scan, k_scan_wide), the
pick step's clamped outputs and the round controller's leaf bounds, tree by tree against the NumPy restatement in monotone_ref.py (grown
by tree_ref.py) on grid gradients and at the bar tree_check.py describes, and the trained models' monotonicity on the engine's own
gradients."""
import numpy as np
import pytest

import tree_check as tc

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- tree by tree against the restatement
def test_numerical_with_nan(built):
    X, g, h, cats = tc.data(1)
    X[:, 2] = -X[:, 2]      # the target falls with this feature: a -1 constraint still lets it split
    model, _ = tc.check_run(X, g, h, cats, 12, 3, mono=[1, 1, -1])
    assert tc.split_features(model) >= {1, 2}


def test_l1_and_max_delta_step(built):
    X, g, h, cats = tc.data(11)
    tc.check_run(X, g, h, cats, 12, 2, mono=[-1, 1, 1], extra="lambda_l1=0.5 lambda_l2=1.0 max_delta_step=0.8")


def test_categoricals_in_constrained_leaves(built):
    X, g, h, cats = tc.data(2, cat=True)
    model, _ = tc.check_run(X, g, h, cats, 16, 3, mono=[1, -1, 1, 0, 0], extra="min_data_per_group=20 cat_smooth=5")
    assert tc.split_features(model) >= {3, 4}, "the case must split on the one-hot and the many-vs-many feature"


def test_wide_features(built):
    """max_bin=511: k_scan_wide's numerical scan under a constraint and a wide categorical feature in constrained leaves"""
    X, g, h, cats = tc.data(4, n=9000, wide=True)
    model, _ = tc.check_run(X, g, h, cats, 12, 2, mono=[1, -1, 0, 1, 0, 0], max_bin=511, extra="min_data_per_group=20 cat_smooth=5")
    assert 3 in tc.split_features(model)


@pytest.mark.parametrize("penalty", [0.5, 2.5])
def test_penalty(built, penalty):
    X, g, h, cats = tc.data(12)
    tc.check_run(X, g, h, cats, 12, 2, mono=[1, -1, 1], penalty=penalty)


def test_extra_trees(built):
    X, g, h, cats = tc.data(13, cat=True)
    tc.check_run(X, g, h, cats, 12, 4, mono=[1, -1, 0, 0, 0], extra="min_data_per_group=20 cat_smooth=5", extra_seed=9)


def test_all_zero_list(built):
    """an all-zero list runs the constrained scans: the restatement's USE_MC scans, gains from the outputs"""
    X, g, h, cats = tc.data(14, cat=True)
    tc.check_run(X, g, h, cats, 12, 2, mono=[0, 0, 0, 0, 0], extra="min_data_per_group=20 cat_smooth=5")


def test_reset_parameter_changes_the_constraints(built):
    X, g, h, cats = tc.data(15)
    model, _ = tc.check_run(X, g, h, cats, 12, 4, mono=[1, 0, 0], reset=(1, tc.mc([-1, -1, 1])))
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


MONO = [1, -1, 1, 0, 0]


@pytest.mark.parametrize("case", sorted(tc.CASES))
def test_predictions_are_monotone(built, case):
    from mmlspark_b200 import capi
    obj, K, label, n = tc.CASES[case]
    X, z = tc.monotone_data(n, 30 + len(case))
    y = label(z)
    group = [20] * (n // 20) if case == "lambdarank" else None
    dsp = tc.DS + " max_bin=255"
    base = "%s num_leaves=31 learning_rate=0.3 min_data_in_leaf=20 verbosity=-1 metric= %s" % (obj, dsp)
    for mono, want_monotone in ((MONO, True), (None, False)):
        params = base + (" " + tc.mc(mono) + " monotone_penalty=0.5" if mono else "")
        model = tc.boost(X, y, params, 8, dsp, group)
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
    X, z = tc.monotone_data(40000, 50)
    dsp = tc.DS + " max_bin=255"
    params = "objective=regression num_leaves=31 learning_rate=0.3 verbosity=-1 metric= tree_learner=data num_machines=2 %s %s" % (tc.mc(MONO), dsp)
    model = tc.boost(X, z, params, 8, dsp, rank_rows=[21000, 19000], port=29700)
    b = capi.Booster(model_str=model)
    try:
        assert _sweep_violations(lambda A: b.predict_device(A, capi.PREDICT_RAW_SCORE), X, MONO, 1) == 0
    finally:
        b.free()


def _two_ranks_match_one(port, device_of=lambda r: 0):
    from mmlspark_b200 import capi  # noqa: F401
    X, g, h, cats = tc.data(6, const_h=True)
    dsp = tc.ds_params(cats, 255)
    params = tc.params(10, "tree_learner=data num_machines=2 monotone_penalty=0.5 " + tc.mc([1, -1, 1]), cats)
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
    single, _ = tc.check_run(X, g, h, cats, 10, 3, mono=[1, -1, 1], penalty=0.5)
    assert tc.trees(res[0]) == tc.trees(single)


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
    g = np.round((-(X[:, 0] * 0.2 + X[:, 3] * 0.1 - X[:, 1] * 0.15 + X[:, 6]) + 0.2 * rng.standard_normal(n)) / tc.GRID) * tc.GRID
    h = tc.grid(rng, 0.5, 1.5, n)
    mono = [1, -1, 0, 1, 0, 0, 1, -1]
    models = []
    for bundle in ("true", "false"):
        dsp = tc.DS + " max_bin=255 enable_bundle=" + bundle
        models.append(tc.run(X, g, h, tc.params(12, tc.mc(mono) + " enable_bundle=" + bundle), 4, dsp))
    assert tc.trees(models[0]) == tc.trees(models[1])
    assert tc.split_features(models[0]) & {0, 1, 3}


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
    X, g, h, cats = tc.data(7, cat=True)
    ds = capi.Dataset.from_mat(X, tc.ds_params(cats, 255)).set_field("label", np.asarray(-g, np.float32))
    try:
        with pytest.raises(Exception) as e:
            capi.Booster(ds, tc.params(8, opts, cats))
        assert msg in str(e.value), str(e.value)
    finally:
        ds.free()


def test_errors_fire_on_every_rank(built):
    """each create-time error and the voting rejection, at create on both ranks, and the voting rejection at ResetParameter"""
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(25, cat=True)
    half = len(X) // 2
    cases = [(o + " tree_learner=data num_machines=2", m) for o, m in ERRORS] + \
            [("monotone_constraints=1,0,0,0,0 tree_learner=voting top_k=2 num_machines=2", "does not support monotone_constraints")]

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
                    b.reset_parameter("monotone_constraints=1,0,0,0,0")
                msgs.append(str(e.value))
                after = b.save_model_to_string()
                b.update_one_iter()
                return msgs, before == after, b.save_model_to_string()
            finally:
                b.free()
        finally:
            ds.free()

    res, errs = tc.on_ranks(2, 29760, body)
    assert not errs, errs
    for msgs, unchanged, model in res:
        for (_, want), got in zip(cases + [(None, "does not support monotone_constraints")], msgs):
            assert want in got, (want, got)
        assert unchanged
        assert "[monotone_constraints: ]" in model and "monotone_constraints=" not in model.split("Tree=")[0]
    assert tc.trees(res[0][2]) == tc.trees(res[1][2])


def test_model_text_round_trips(built):
    from mmlspark_b200 import capi
    X, g, h, cats = tc.data(8)
    dsp = tc.ds_params(cats, 255)
    model = tc.run(X, g, h, tc.params(8, "mc=1,-1,0 monotone_constraints_method=basic ms_penalty=1.5", cats), 2, dsp)
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
    plain = tc.run(X, g, h, tc.params(8, "", cats), 2, dsp)
    assert "monotone_constraints=" not in plain.split("Tree=")[0]
    assert "[monotone_constraints: ]" in plain and "[monotone_penalty: 0]" in plain


def test_estimator(built):
    """LightGBMRegressor(monotoneConstraints=...) trains the model of the low-level run with its parameter string"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.params import dataset_params
    X, z = tc.monotone_data(5000, 10)
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
    assert tc.trees(model) == tc.trees(low)
    assert "monotone_constraints=1 -1 1 0 0" in model
