"""LGBM_BoosterRefit on the device against the NumPy restatement (refit_ref): every leaf of every tree and the final training scores, the
structure left as it was, the predictors, save and reload, the staging in several batches and row blocks, the global-atomic path of large
trees, data-parallel rank-threads, the checks (a failed refit changes nothing) and capi.refit.

Bars: l2 regression within 4 fp64 ulps in every iteration (its gradient is one fp64 subtract cast to float, which NumPy repeats); every
objective's first iteration within 4 ulps, on the engine's gradients read just before the refit; later iterations of the other objectives
1e-9 relative (their gradients go through exp)."""
import numpy as np
import pytest

import refit_ref as R
import tree_check as TC

pytestmark = pytest.mark.gpu

DS = "max_bin=63 min_data_in_bin=3 bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 min_data_in_leaf=10 learning_rate=0.1 verbosity=-1 " + DS
STRUCTURE = ("split_feature", "threshold", "decision_type", "left_child", "right_child", "leaf_count", "internal_count", "leaf_weight",
             "internal_value", "internal_weight")


@pytest.fixture(scope="module")
def capi(built):
    from mmlspark_b200 import capi as c
    c.load()
    return c


def _data(n, seed, objective="regression", K=3):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 6))
    z = X[:, 0] + np.sin(2 * X[:, 1]) + 0.5 * X[:, 2] * X[:, 3] + 0.2 * rng.standard_normal(n)
    if objective == "binary":
        y = (z > np.median(z)).astype(np.float32)
    elif objective == "multiclass":
        y = np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])).astype(np.float32)
    elif objective == "lambdarank":
        y = np.digitize(z, np.quantile(z, [0.5, 0.8, 0.95])).astype(np.float32)
    else:
        y = z.astype(np.float32)
    return X, y


def _dataset(capi, X, y, w=None, init=None, group=None):
    ds = capi.Dataset.from_mat(X, DS).set_field("label", y)
    if w is not None:
        ds.set_field("weight", w)
    if init is not None:
        ds.set_field("init_score", init)
    if group is not None:
        ds.set_field("group", group)
    return ds


def _train(capi, X, y, params, iters, **fields):
    ds = _dataset(capi, X, y, **fields)
    b = capi.Booster(ds, params)
    try:
        for _ in range(iters):
            b.update_one_iter()
        return b.save_model_to_string()
    finally:
        b.free(); ds.free()


def _leaf(capi, model, X):
    old = capi.Booster(model_str=model)
    try:
        return old.predict_for_mat(X, capi.PREDICT_LEAF_INDEX).astype(np.int32)
    finally:
        old.free()


def _merged(capi, model, X, y, params, decay, **fields):
    """steps 2 and 3 of the refit flow: a booster on X with the model merged into it; returns (booster, dataset)"""
    ds = _dataset(capi, X, y, **fields)
    b = capi.Booster(ds, "%s refit_decay_rate=%r" % (params, decay))
    old = capi.Booster(model_str=model)
    b.merge(old)
    old.free()
    return b, ds


def _opts(params):
    kv = dict(t.split("=", 1) for t in params.split())
    return dict(l1=float(kv.get("lambda_l1", 0)), l2=float(kv.get("lambda_l2", 0)), max_delta_step=float(kv.get("max_delta_step", 0)),
                path_smooth=float(kv.get("path_smooth", 0)))


def _check(got_model, model, new, K, exact_iters):
    """the refit model's trees against the model it started from (structure, shrinkage) and refit_ref's leaf values; the first
    exact_iters iterations within 4 ulps, the rest within 1e-9"""
    from mmlspark_b200.modeltext import parse_model
    got, was = parse_model(got_model)["trees"], parse_model(model)["trees"]
    assert len(got) == len(was) == len(new)
    for m, (t, o, v) in enumerate(zip(got, was, new)):
        assert t["num_leaves"] == o["num_leaves"] and t.get("shrinkage") == o.get("shrinkage"), m
        for k in STRUCTURE:
            if k in o:
                assert np.array_equal(t[k], o[k]), (m, k)
        if m // K < exact_iters:
            assert (TC.ulps(t["leaf_value"], v) <= 4).all(), (m, t["leaf_value"], v)
        else:
            np.testing.assert_allclose(t["leaf_value"], v, rtol=1e-9, atol=1e-300, err_msg="model %d" % m)


CASES = {
    "l2": ("objective=regression", {}),
    "l2_weight": ("objective=regression", {"w": True}),
    "l2_init": ("objective=regression", {"init": True}),
    "l2_l1_mds": ("objective=regression lambda_l1=0.5 lambda_l2=1 max_delta_step=0.3", {}),
    "l2_smooth": ("objective=regression path_smooth=5", {}),
    "l2_no_average": ("objective=regression boost_from_average=false", {}),
    "binary": ("objective=binary", {}),
    "multiclass": ("objective=multiclass num_class=3", {}),
    "dart": ("objective=regression boosting=dart drop_rate=0.3", {}),
    "goss": ("objective=regression boosting=goss learning_rate=0.5 top_rate=0.3 other_rate=0.2", {}),
}


@pytest.mark.parametrize("decay", [0.0, 0.5, 0.9])
@pytest.mark.parametrize("case", sorted(CASES))
def test_refit_matches_reference(capi, case, decay):
    params, f = CASES[case]
    params = BASE + " " + params
    objective = params.split("objective=")[1].split()[0]
    K = 3 if objective == "multiclass" else 1
    X, y = _data(4000, 1, objective)
    rng = np.random.default_rng(2)
    w = rng.uniform(0.5, 2.0, len(y)).astype(np.float32) if f.get("w") else None
    init = rng.uniform(-1, 1, len(y)) if f.get("init") else None
    model = _train(capi, X, y, params, 8, w=w, init=init)
    # the refit data: new rows from the same distribution, labels shifted
    X2, y2 = _data(3000, 3, objective)
    if objective == "regression":
        y2 = (y2 + 0.5).astype(np.float32)
    w2 = rng.uniform(0.5, 2.0, len(y2)).astype(np.float32) if f.get("w") else None
    init2 = rng.uniform(-1, 1, len(y2)) if f.get("init") else None
    leaf = _leaf(capi, model, X2)
    b, ds = _merged(capi, model, X2, y2, params, decay, w=w2, init=init2)
    try:
        g0 = b.get_gradients()
        b.refit(leaf)
        from mmlspark_b200.modeltext import parse_model
        trees = parse_model(model)["trees"]
        l2 = objective == "regression"
        new, score = R.refit(trees, K, leaf, y2, objective, decay, w=w2, init_score=init2, num_class=K, first_grads=None if l2 else g0,
                             **_opts(params))
        _check(b.save_model_to_string(), model, new, K, len(trees) // K if l2 else 1)
        np.testing.assert_allclose(b.get_scores(), score, rtol=1e-12 if l2 else 1e-9, atol=1e-12)
    finally:
        b.free(); ds.free()


@pytest.mark.parametrize("decay", [0.0, 0.9])
def test_refit_own_trained_model(capi, decay):
    """a booster refits the model it trained itself, from its current training scores"""
    X, y = _data(4000, 5)
    params = BASE + " objective=regression refit_decay_rate=%r" % decay
    ds = _dataset(capi, X, y)
    b = capi.Booster(ds, params)
    try:
        for _ in range(6):
            b.update_one_iter()
        model = b.save_model_to_string()
        leaf = b.predict_for_mat(X, capi.PREDICT_LEAF_INDEX).astype(np.int32)
        s0 = b.get_scores()
        b.refit(leaf)
        from mmlspark_b200.modeltext import parse_model
        new, score = R.refit(parse_model(model)["trees"], 1, leaf, y, "regression", decay, init_score=s0)
        _check(b.save_model_to_string(), model, new, 1, 6)
        np.testing.assert_allclose(b.get_scores(), score, rtol=1e-12, atol=1e-12)
    finally:
        b.free(); ds.free()


def test_lambdarank_scores_equal_raw_predictions(capi):
    X, y = _data(3000, 7, "lambdarank")
    group = np.full(30, 100, np.int32)
    params = BASE + " objective=lambdarank"
    model = _train(capi, X, y, params, 5, group=group)
    leaf = _leaf(capi, model, X)
    b, ds = _merged(capi, model, X, y, params, 0.5, group=group)
    try:
        b.refit(leaf)
        np.testing.assert_allclose(b.get_scores(), b.predict_for_mat(X, capi.PREDICT_RAW_SCORE).ravel(), rtol=1e-12, atol=1e-12)
    finally:
        b.free(); ds.free()


def test_decay_one_keeps_every_leaf(capi):
    X, y = _data(3000, 9)
    params = BASE + " objective=regression"
    model = _train(capi, X, y, params, 6)
    b, ds = _merged(capi, model, X, y, params, 1.0)
    try:
        before = b.save_model_to_string()
        b.refit(_leaf(capi, model, X))
        after = b.save_model_to_string()
        assert TC.trees(after) == TC.trees(before)
        assert "[refit_decay_rate: 1]" in after
    finally:
        b.free(); ds.free()


def test_predictors_save_and_reload(capi):
    X, y = _data(3000, 11)
    params = BASE + " objective=regression"
    model = _train(capi, X, y, params, 6)
    b, ds = _merged(capi, model, X, (y + 1).astype(np.float32), params, 0.5)
    try:
        before = b.predict_device(X, capi.PREDICT_RAW_SCORE)
        b.refit(_leaf(capi, model, X))
        host = b.predict_for_mat(X, capi.PREDICT_RAW_SCORE).ravel()
        dev = b.predict_device(X, capi.PREDICT_RAW_SCORE).ravel()
        assert np.array_equal(host, dev) and not np.array_equal(dev, before.ravel())      # the device forest sees the new leaves
        np.testing.assert_allclose(b.get_predict(0), host, rtol=1e-12, atol=1e-12)
        text = b.save_model_to_string()
        assert "[refit_decay_rate: 0.5]" in text
        again = capi.Booster(model_str=text)
        assert np.array_equal(again.predict_for_mat(X, capi.PREDICT_RAW_SCORE).ravel(), host)
        again.free()
    finally:
        b.free(); ds.free()


def _refit_model(capi, model, X, y, params, decay, leaf=None):
    b, ds = _merged(capi, model, X, y, params, decay)
    try:
        b.refit(_leaf(capi, model, X) if leaf is None else leaf)
        return b.save_model_to_string(), b.get_scores(), b.refit_timing()
    finally:
        b.free(); ds.free()


def test_staging_batches_and_row_blocks_are_bit_identical(capi, monkeypatch):
    X, y = _data(5000, 13, "multiclass")
    params = BASE + " objective=multiclass num_class=3"
    model = _train(capi, X, y, params, 5)
    one, s1, t1 = _refit_model(capi, model, X, y, params, 0.3)
    assert t1["batches"] == 1
    monkeypatch.setenv("B200GBM_REFIT_STAGING", "2,1000")      # two models per batch, 1000-row blocks
    many, s2, t2 = _refit_model(capi, model, X, y, params, 0.3)
    assert t2["batches"] == 8 and t2["blocks"] == 8 * 5, t2
    assert TC.trees(many) == TC.trees(one) and np.array_equal(s1, s2)


def test_large_tree_uses_global_atomics(capi):
    rng = np.random.default_rng(17)
    n = 20000
    X = rng.standard_normal((n, 6))
    y = (X[:, 0] + rng.standard_normal(n)).astype(np.float32)
    params = "objective=regression num_leaves=6000 min_data_in_leaf=1 min_sum_hessian_in_leaf=0 max_bin=255 verbosity=-1 num_threads=0"
    model = _train(capi, X, y, params, 2)
    from mmlspark_b200.modeltext import parse_model
    trees = parse_model(model)["trees"]
    assert max(t["num_leaves"] for t in trees) > 4096
    leaf = _leaf(capi, model, X)
    got, score, _ = _refit_model(capi, model, X, (y * 0.5).astype(np.float32), params, 0.2, leaf)
    new, ref_score = R.refit(trees, 1, leaf, (y * 0.5).astype(np.float32), "regression", 0.2)
    _check(got, model, new, 1, 2)
    np.testing.assert_allclose(score, ref_score, rtol=1e-12, atol=1e-12)


def _tree_text(model):
    return model[model.index("Tree=0"):].split("\nparameters:")[0]


@pytest.mark.parametrize("R_", [2, 3])
def test_ranks_equal_one_rank_over_all_rows(capi, R_):
    X, y = _data(6000, 19)
    params = BASE + " objective=regression"
    model = _train(capi, X, y, params, 5)
    leaf = _leaf(capi, model, X)
    one, _, _ = _refit_model(capi, model, X, y, params, 0.4, leaf)
    offs = np.linspace(0, len(X), R_ + 1).astype(int)

    def body(r):
        sl = slice(offs[r], offs[r + 1])
        b, ds = _merged(capi, model, X[sl], y[sl], params, 0.4)
        try:
            b.refit(np.ascontiguousarray(leaf[sl]))
            return b.save_model_to_string()
        finally:
            b.free(); ds.free()

    out, errs = TC.on_ranks(R_, 14100 + 10 * R_, body)
    assert not errs, errs
    for text in out:      # the trees; the header's feature ranges are each rank's own
        assert _tree_text(text) == _tree_text(one)


def _unchanged(b, X):
    return b.save_model_to_string(), b.get_scores(), b.predict_for_mat(X, 1), b.predict_device(X, 1)


def _assert_same(a, b):
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x, y)


def test_failed_refit_changes_nothing(capi, monkeypatch):
    X, y = _data(3000, 23)
    params = BASE + " objective=regression"
    model = _train(capi, X, y, params, 6)
    leaf = _leaf(capi, model, X)
    from mmlspark_b200.modeltext import parse_model
    num_leaves = [t["num_leaves"] for t in parse_model(model)["trees"]]
    # a prediction-only booster
    p = capi.Booster(model_str=model)
    with pytest.raises(capi.LightGBMError, match="training booster"):
        p.refit(leaf)
    p.free()
    # decay outside [0, 1]
    for d in (-0.1, 1.5):
        b, ds = _merged(capi, model, X, y, params, d)
        before = _unchanged(b, X)
        with pytest.raises(capi.LightGBMError, match=r"refit_decay_rate should be in \[0, 1\]"):
            b.refit(leaf)
        _assert_same(before, _unchanged(b, X))
        b.free(); ds.free()
    b, ds = _merged(capi, model, X, y, params, 0.5)
    before = _unchanged(b, X)
    bad_rows = leaf[:-1]
    with pytest.raises(capi.LightGBMError, match="2999 rows, the training data has 3000"):
        b.refit(bad_rows)
    with pytest.raises(capi.LightGBMError, match="5 columns, the booster has 6 models"):
        b.refit(leaf[:, :-1])
    hi = leaf.copy()
    hi[5, 3] = num_leaves[3]
    with pytest.raises(capi.LightGBMError, match=r"leaf_preds\[5\]\[3\] = %d is outside \[0, %d\)" % (num_leaves[3], num_leaves[3])):
        b.refit(hi)
    neg = leaf.copy()
    neg[7, 2] = -1
    neg[9, 1] = -5      # later in row-major order: the first one is named
    with pytest.raises(capi.LightGBMError, match=r"leaf_preds\[7\]\[2\] = -1 is outside"):
        b.refit(neg)
    # a bad index in the last batch of models, after earlier batches changed the scores: they are restored
    monkeypatch.setenv("B200GBM_REFIT_STAGING", "1,700")
    late = leaf.copy()
    late[100, 5] = num_leaves[5] + 1
    with pytest.raises(capi.LightGBMError, match=r"leaf_preds\[100\]\[5\]"):
        b.refit(late)
    assert b.refit_timing()["batches"] == 6
    _assert_same(before, _unchanged(b, X))
    b.free(); ds.free()


def test_custom_objective_and_rf_fail(capi):
    X, y = _data(3000, 29)
    ds = _dataset(capi, X, y)
    b = capi.Booster(ds, BASE + " objective=regression")
    g = np.zeros(len(y), np.float32) + 0.5
    b.update_one_iter_custom(g, np.ones(len(y), np.float32))
    model = b.save_model_to_string()
    before = _unchanged(b, X)
    with pytest.raises(capi.LightGBMError, match="No object function provided"):
        b.refit(_leaf(capi, model, X))
    _assert_same(before, _unchanged(b, X))
    b.free()
    r = capi.Booster(ds, BASE + " objective=regression boosting=rf bagging_fraction=0.7 bagging_freq=1")
    for _ in range(3):
        r.update_one_iter()
    model = r.save_model_to_string()
    before = _unchanged(r, X)
    with pytest.raises(capi.LightGBMError, match="boosting=rf does not support refit"):
        r.refit(_leaf(capi, model, X))
    _assert_same(before, _unchanged(r, X))
    r.free(); ds.free()


def test_one_bad_rank_fails_every_rank(capi):
    X, y = _data(4000, 31)
    params = BASE + " objective=regression"
    model = _train(capi, X, y, params, 4)
    leaf = _leaf(capi, model, X)

    def body(r):
        sl = slice(2000 * r, 2000 * (r + 1))
        mine = np.ascontiguousarray(leaf[sl])
        if r == 1:
            mine[10, 1] = -1
        b, ds = _merged(capi, model, X[sl], y[sl], params, 0.5)
        try:
            before = b.get_scores()
            try:
                b.refit(mine)
            finally:
                assert np.array_equal(b.get_scores(), before)
        finally:
            b.free(); ds.free()

    out, errs = TC.on_ranks(2, 14200, body)
    msgs = dict(errs)
    assert set(msgs) == {0, 1}, errs
    assert "another rank's leaf_preds failed" in msgs[0] and "leaf_preds[10][1] = -1" in msgs[1]


def test_capi_refit_equals_the_four_steps(capi):
    X, y = _data(3000, 37, "binary")
    params = BASE + " objective=binary"
    model = _train(capi, X, y, params, 5)
    X2, y2 = _data(2500, 41, "binary")
    w = np.random.default_rng(43).uniform(0.5, 2, len(y2)).astype(np.float32)
    b = capi.refit(model, X2, y2, params, decay_rate=0.6, weight=w)
    got = b.save_model_to_string()
    ds_keep = b.train_set
    b.free(); ds_keep.free()
    m, ds = _merged(capi, model, X2, y2, params, 0.6, w=w)
    m.refit(_leaf(capi, model, X2))
    assert got == m.save_model_to_string()
    m.free(); ds.free()
