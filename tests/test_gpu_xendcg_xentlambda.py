"""rank_xendcg and cross_entropy_lambda objectives (k_grad_xendcg, k_grad_xentlambda) and the cross_entropy_lambda and kullback_leibler
metrics on the device, against the NumPy restatement in tests/xendcg_xentlambda_ref.py.

Gradients are read with B200GBM_BoosterGetGradients at chosen scores.  Bar as test_gpu_gradients.py: non-finite values at the same
positions with the same kind, finite values within 1 float32 ulp, at least 99.9 % bit-equal.  rank_xendcg's lambda is a float sum of
three terms that can cancel, so its ulp is taken at max(|f32 t1|, |f32 t2|, |f32 t3|).  Training parity: the built-in objective
against the same engine fed the NumPy gradients through LGBM_BoosterUpdateOneIterCustom, at the bar of test_gpu_parity.py."""
import threading
import zlib

import numpy as np
import pytest

import xendcg_xentlambda_ref as R
from test_gpu_multi import _ngpu, _params as _multi_params

pytestmark = pytest.mark.gpu

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 learning_rate=0.1 min_data_in_leaf=20 verbosity=-1 "
GRID = np.array([0.0, -0.0, 1e-300, -1e-300, 1e-8, -1e-8, 0.5, -0.5, 5.0, -5.0, 30.0, -30.0, 37.0, -37.0, 700.0, -700.0,
                 709.7, -709.7, 710.0, -710.0, 745.0, -745.0, 800.0, -800.0])


def _ordered(a):
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7FFFFFFF) - 1, b)


def _compare(got, want, what, scale=None):
    """the module's bar; scale: the magnitude whose float32 ulp bounds |got - want| (default: want itself, i.e. 1 ulp)"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, what
    fg, fw = np.isfinite(got), np.isfinite(want)
    bad = np.nonzero(fg != fw)[0]
    assert len(bad) == 0, "%s: finite / non-finite differ at %d positions, first %d: got %r want %r" % (what, len(bad), bad[0], got[bad[0]], want[bad[0]])
    nf = ~fw
    assert np.array_equal(np.isnan(got[nf]), np.isnan(want[nf])), what + ": inf where NaN is expected or the reverse"
    assert np.array_equal(got[np.isinf(want)], want[np.isinf(want)]), what + ": infinities of the wrong sign"
    if scale is None:
        d = np.abs(_ordered(got[fw]) - _ordered(want[fw]))
        assert d.max(initial=0) <= 1, "%s: %d ulps apart" % (what, d.max())
    else:
        sc = np.asarray(scale, np.float32)[fw]
        err = np.abs(got[fw].astype(np.float64) - want[fw].astype(np.float64))
        lim = np.spacing(np.abs(sc).astype(np.float32)).astype(np.float64)
        i = np.argmax(err - lim) if len(err) else 0
        assert (err <= lim).all(), "%s: |got - want| %r above the ulp %r of the scale at %d" % (what, err[i], lim[i], i)
    not_equal = int((got[fw].view(np.int32) != want[fw].view(np.int32)).sum())
    assert not_equal <= 0.001 * got.size, "%s: %d of %d elements are not bit-equal" % (what, not_equal, got.size)
    return not_equal


def _booster(X, y, params, weight=None, group=None, init_score=None):
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    for name, arr in (("weight", weight), ("group", group), ("init_score", init_score)):
        if arr is not None:
            ds.set_field(name, arr)
    return capi.Booster(ds, BASE + params), ds


# ------------------------------------------------------------------------------------------------ cross_entropy_lambda gradients
@pytest.mark.parametrize("wmode", ["none", "uniform", "wide"])
def test_xentlambda_gradients_match_numpy(built, wmode):
    rng = np.random.default_rng(zlib.crc32(wmode.encode()))
    n = 200_003
    s = 3.0 * rng.standard_normal(n)
    pick = rng.random(n) < 0.5
    s[pick] = GRID[rng.integers(0, len(GRID), int(pick.sum()))]
    s[:len(GRID)] = GRID
    u = rng.random(n)
    y = np.where(u < 0.25, 0.0, np.where(u < 0.5, 1.0, rng.random(n))).astype(np.float32)
    w = None if wmode == "none" else (np.full(n, 0.75, np.float32) if wmode == "uniform" else (10.0 ** rng.uniform(-20.0, 20.0, n)).astype(np.float32))
    b, _ = _booster(rng.standard_normal((n, 2)), y, "objective=xentlambda", weight=w, init_score=s)
    g, h = b.get_gradients()
    rg, rh = R.xentlambda_gradients(s, y, w)
    keep = np.ones(n, bool)
    if w is not None:
        # [UPSTREAM] computes z = 1 - exp(-x), x = w log1p(e^s), which keeps only log2(x) + 53 bits of z; the hessian cancels once
        # more in 1 + w e^s - 1 / (1 - z).  For x < 2^-8 the last bit of exp, where the device may differ from the host, moves the
        # float results (at x near 1e-16 it decides between z = 0, a non-finite gradient, and a finite one), so those rows are not
        # compared.  Below x = 2^-60 both sides round exp(-x) to 1 and agree again.
        with np.errstate(all="ignore"):
            x = w.astype(np.float64) * np.log1p(np.exp(s))
        keep = ~((x >= 2.0 ** -60) & (x < 2.0 ** -8))
        assert keep.mean() > 0.5
    _compare(g[keep], rg[keep], "grad")
    _compare(h[keep], rh[keep], "hess")


def test_xentlambda_rejects_non_positive_weights_and_labels_outside_01(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(2)
    X, y = rng.standard_normal((500, 3)), rng.random(500).astype(np.float32)
    w = (0.5 + rng.random(500)).astype(np.float32)
    w[17] = 0.0
    with pytest.raises(capi.LightGBMError, match="non-positive"):
        _booster(X, y, "objective=cross_entropy_lambda", weight=w)
    y[3] = 1.5
    with pytest.raises(capi.LightGBMError, match="outside"):
        _booster(X, y, "objective=cross_entropy_lambda")


# ------------------------------------------------------------------------------------------------ rank_xendcg gradients
def _rank_data(rng, sizes, max_label=4):
    n = int(np.sum(sizes))
    X = rng.standard_normal((n, 6))
    rel = np.clip(np.round(X[:, 0] + 0.5 * X[:, 1] + 0.5 * rng.standard_normal(n) + 1.5), 0, 4)
    if max_label > 4:
        rel = np.where(rng.random(n) < 0.05, rng.integers(0, max_label + 1, n), rel)
    return X, rel.astype(np.float32)


XE_CASES = [("labels0-4", {}, 4, False), ("labels0-30-weighted", {}, 30, True), ("seed7", {"objective_seed": 7}, 4, False)]


@pytest.mark.parametrize("case", XE_CASES, ids=[c[0] for c in XE_CASES])
def test_xendcg_gradients_match_numpy_before_and_after_iterations(built, case):
    name, extra, max_label, weighted = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    sizes = np.concatenate([[1, 2, 100, 3000, 20_500, 1], rng.integers(2, 60, 400)]).astype(np.int32)
    X, y = _rank_data(rng, sizes, max_label)
    n = len(y)
    w = (0.25 + 2 * rng.random(n)).astype(np.float32) if weighted else None
    seed = extra.get("objective_seed", 5)
    b, _ = _booster(X, y, "objective=rank_xendcg " + " ".join("%s=%s" % kv for kv in extra.items()), weight=w, group=sizes)
    rands = R.xendcg_rands(len(sizes), seed)

    def check(when):
        s = b.get_scores()
        g, h = b.get_gradients()
        g2, h2 = b.get_gradients()          # reading does not advance the random states
        assert np.array_equal(g.view(np.int32), g2.view(np.int32)) and np.array_equal(h.view(np.int32), h2.view(np.int32))
        rg, rh, scale = R.xendcg_gradients(s, y, sizes, rands, w)       # takes the draws the next iteration trains on
        _compare(h, rh, "%s %s hess" % (name, when))
        _compare(g, rg, "%s %s grad" % (name, when), scale=scale)

    check("before iteration 0")
    b.update_one_iter()
    check("after 1 iteration")
    b.update_one_iter()
    R.xendcg_gradients(b.get_scores(), y, sizes, rands, w)             # the third iteration's draws
    b.update_one_iter()
    check("after 3 iterations")


def test_xendcg_saturated_softmax_gives_the_reference_non_finite_pattern(built):
    rng = np.random.default_rng(8)
    sizes = np.concatenate([[10, 6, 40], np.full(100, 30)]).astype(np.int32)      # enough rows for the bit-equal share
    X, y = _rank_data(rng, sizes)
    s = rng.standard_normal(len(y))
    s[0], s[1] = 800.0, -800.0                # query 0: rho = 1 at document 0, exactly 0 elsewhere
    s[10:16] = [900.0, 900.0, -900.0, 0.0, 1.0, 2.0]
    b, _ = _booster(X, y, "objective=rank_xendcg", group=sizes, init_score=s)
    g, h = b.get_gradients()
    rg, rh, scale = R.xendcg_gradients(s, y, sizes, R.xendcg_rands(len(sizes)))
    assert not np.isfinite(rg).all()
    _compare(h, rh, "hess")
    _compare(g, rg, "grad", scale=scale)


# ------------------------------------------------------------------------------------------------ training parity
def _parity(X, y, params, grad_fn, iters, weight=None, group=None):
    """the built-in objective against the same booster settings fed grad_fn(scores) through the custom-gradient path"""
    from mmlspark_b200.modeltext import compare_models, parse_model
    b1, _ = _booster(X, y, params, weight=weight, group=group)
    b2, _ = _booster(X, y, params, weight=weight, group=group)
    for _ in range(iters):
        f1 = b1.update_one_iter()
        g, h = grad_fn(b2.get_scores())
        f2 = b2.update_one_iter_custom(g, h)
        assert f1 == f2
    m1, m2 = parse_model(b1.save_model_to_string()), parse_model(b2.save_model_to_string())
    compare_models(m1, m2)
    np.testing.assert_allclose(b1.get_scores(), b2.get_scores(), rtol=0, atol=1e-9)
    return m1


@pytest.mark.parametrize("weighted", [False, True])
def test_xentlambda_training_parity(built, weighted):
    rng = np.random.default_rng(21 + weighted)
    n = 40_000
    X = rng.standard_normal((n, 10))
    y = (1.0 / (1.0 + np.exp(-(X[:, 0] - 0.5 * X[:, 1] + 0.3 * rng.standard_normal(n))))).astype(np.float32)
    w = (0.2 + 2.0 * rng.random(n)).astype(np.float32) if weighted else None
    _parity(X, y, "objective=cross_entropy_lambda boost_from_average=false", lambda s: R.xentlambda_gradients(s, y, w), 30, weight=w)


def test_xentlambda_init_score(built):
    """boost_from_average: the first tree of a booster that cannot split is the constant log(expm1(weighted label mean))"""
    from mmlspark_b200.modeltext import parse_model
    rng = np.random.default_rng(23)
    n = 5000
    X, y = rng.standard_normal((n, 3)), rng.random(n).astype(np.float32)
    w = (0.5 + rng.random(n)).astype(np.float32)
    b, _ = _booster(X, y, "objective=cross_entropy_lambda min_data_in_leaf=%d" % n, weight=w)
    b.update_one_iter()
    tree = parse_model(b.save_model_to_string())["trees"][0]
    assert tree["num_leaves"] == 1
    np.testing.assert_allclose(tree["leaf_value"], R.xentlambda_init_score(y, w), rtol=1e-12)


def test_xendcg_training_parity_and_seeds(built):
    rng = np.random.default_rng(31)
    sizes = rng.integers(2, 40, 600).astype(np.int32)
    X, y = _rank_data(rng, sizes)
    models = []
    for seed in (5, 7):
        rands = R.xendcg_rands(len(sizes), seed)
        m = _parity(X, y, "objective=rank_xendcg objective_seed=%d" % seed, lambda s: R.xendcg_gradients(s, y, sizes, rands)[:2], 30, group=sizes)
        assert m["header"]["objective"] == "rank_xendcg"
        models.append(m)
    assert any(not np.array_equal(a["leaf_value"], b["leaf_value"]) for a, b in zip(models[0]["trees"], models[1]["trees"]))


# ------------------------------------------------------------------------------------------------ metrics
def _transform(objective, raw):
    if objective == "cross_entropy_lambda":
        return np.log1p(np.exp(raw))
    return 1.0 / (1.0 + np.exp(-raw))         # binary (sigmoid 1) and cross_entropy


@pytest.mark.parametrize("objective", ["cross_entropy_lambda", "cross_entropy", "binary"])
@pytest.mark.parametrize("weighted", [False, True])
def test_metrics_match_numpy(built, objective, weighted):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(41 + weighted)
    n, nv = 30_000, 7_000
    X = rng.standard_normal((n, 6))
    y = (1.0 / (1.0 + np.exp(-(X[:, 0] + 0.5 * rng.standard_normal(n))))).astype(np.float32)
    if objective == "binary":
        y = (y > 0.5).astype(np.float32)
    w = (0.2 + 2.0 * rng.random(n)).astype(np.float32) if weighted else None
    init = 0.5 * rng.standard_normal(n)
    metric = "xentlambda,kldiv" if weighted else "cross_entropy_lambda,kullback_leibler"
    b, ds = _booster(X, y, "objective=%s metric=%s" % (objective, metric), weight=w, init_score=init)
    dv = capi.Dataset.from_mat(X[:nv] + 0.1, DS_PARAMS, reference=ds).set_field("label", y[:nv])
    if weighted:
        dv.set_field("weight", w[:nv])
    b.add_valid(dv)
    assert b.eval_names() == ["cross_entropy_lambda", "kullback_leibler"]
    for _ in range(3):
        b.update_one_iter()
    for idx, (yy, ww) in enumerate(((y, w), (y[:nv], None if w is None else w[:nv]))):
        p = _transform(objective, b.get_scores(idx))
        got = b.get_eval(idx)
        np.testing.assert_allclose(got[0], R.metric_xentlambda(p, yy, ww), rtol=1e-10)
        np.testing.assert_allclose(got[1], R.metric_kldiv(p, yy, ww), rtol=1e-10)


def test_metrics_reject_bad_labels_and_weights(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(43)
    X = rng.standard_normal((600, 3))
    y = rng.random(600).astype(np.float32)
    bad = y.copy()
    bad[5] = -0.5
    for m in ("cross_entropy_lambda", "kullback_leibler"):
        with pytest.raises(capi.LightGBMError, match="outside"):
            _booster(X, bad, "objective=regression metric=" + m)
    w = np.zeros(600, np.float32)
    with pytest.raises(capi.LightGBMError, match="sum of weights is zero"):
        _booster(X, y, "objective=regression metric=kldiv", weight=w)
    w[:] = 1.0
    w[9] = -1.0
    with pytest.raises(capi.LightGBMError, match="negative"):
        _booster(X, y, "objective=regression metric=kldiv", weight=w)
    b, ds = _booster(X, y, "objective=regression metric=kldiv")
    dv = capi.Dataset.from_mat(X, DS_PARAMS, reference=ds).set_field("label", bad)
    with pytest.raises(capi.LightGBMError, match="outside"):
        b.add_valid(dv)


# ------------------------------------------------------------------------------------------------ model text, estimators
def test_xentlambda_model_round_trip(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(51)
    n = 20_000
    X = rng.standard_normal((n, 8))
    y = (1.0 / (1.0 + np.exp(-X[:, 0]))).astype(np.float32)
    b, _ = _booster(X, y, "objective=cross_entropy_lambda")
    for _ in range(10):
        b.update_one_iter()
    text = b.save_model_to_string()
    assert "objective=cross_entropy_lambda" in text
    loaded = capi.Booster(model_str=text)
    for row in X[:5]:
        raw = loaded.predict_for_mat_single(row, capi.PREDICT_RAW_SCORE)[0]
        np.testing.assert_allclose(loaded.predict_for_mat_single(row)[0], np.log1p(np.exp(raw)), rtol=1e-12)
    host = loaded.predict_for_mat(X[:3000])
    np.testing.assert_allclose(loaded.predict_device(X[:3000]).reshape(host.shape), host, rtol=0, atol=1e-12)


def test_ranker_estimator_with_rank_xendcg(built):
    from mmlspark_b200.lightgbm import Frame, LightGBMRanker
    rng = np.random.default_rng(61)
    sizes = rng.integers(5, 30, 400)
    q = np.repeat(np.arange(400), sizes)
    X, rel = _rank_data(rng, sizes)
    df = Frame({"features": X, "label": rel.astype(np.float64), "query": q})
    m = LightGBMRanker(groupCol="query", objective="rank_xendcg", numIterations=20, numTasks=1, minDataInLeaf=5).fit(df)
    assert "objective=rank_xendcg" in m.getNativeModel()
    assert np.corrcoef(m.transform(df)["prediction"], df["label"])[0, 1] > 0.5
    shap = m.getFeatureShaps(df["features"][0])
    assert abs(sum(shap) - m.predict(df["features"][0])) < 1e-9


def test_regressor_estimator_with_xentlambda_and_kullback_leibler_early_stopping(built):
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    rng = np.random.default_rng(71)
    n = 20_000
    X = rng.standard_normal((n, 6))
    y = 1.0 / (1.0 + np.exp(-(2 * X[:, 0] + 0.5 * rng.standard_normal(n))))
    df = Frame({"features": X, "label": y, "valid": rng.random(n) < 0.25})
    m = LightGBMRegressor(objective="cross_entropy_lambda", metric="kullback_leibler", validationIndicatorCol="valid",
                          earlyStoppingRound=3, numIterations=400, learningRate=0.3, numTasks=1).fit(df)
    assert "objective=cross_entropy_lambda" in m.getNativeModel()
    assert m.getBoosterNumTotalIterations() < 400              # stopped early on the validation divergence
    pred = m.transform(df)["prediction"]
    assert np.corrcoef(pred, y)[0, 1] > 0.9


def test_reset_parameter_checks_the_new_metrics(built):
    """LGBM_BoosterResetParameter applies the checks of booster creation and AddValidData to the metrics it names; a rejected reset
    leaves the booster's metrics as they were"""
    from mmlspark_b200 import capi
    rng = np.random.default_rng(45)
    X = rng.standard_normal((2000, 4))
    y = rng.random(2000).astype(np.float32)
    b, ds = _booster(X, y, "objective=regression metric=l2")
    b.update_one_iter()
    b.reset_parameter("metric=kldiv,xentlambda")
    assert b.eval_names() == ["kullback_leibler", "cross_entropy_lambda"]
    bad = y[:500].copy()
    bad[7] = 2.0
    b2, ds2 = _booster(X, y, "objective=regression metric=l2")
    b2.add_valid(capi.Dataset.from_mat(X[:500], DS_PARAMS, reference=ds2).set_field("label", bad))
    with pytest.raises(capi.LightGBMError, match="outside"):
        b2.reset_parameter("metric=kullback_leibler")
    assert b2.eval_names() == ["l2"]
    b2.update_one_iter()
    assert np.isfinite(b2.get_eval(1)).all()


# ------------------------------------------------------------------------------------------------ two ranks
def _run_two_ranks(X, y, groups, params, iters, base_port, grad_fn=None, weight=None):
    """R rank-threads in one process as test_gpu_multi.run_ranks, each with its rows (and query groups: groups[r], None without).
    grad_fn(r, scores) -> (g, h) trains through LGBM_BoosterUpdateOneIterCustom instead of the built-in objective."""
    from mmlspark_b200 import capi
    R = len(groups)
    rows = [int(np.sum(g)) for g in groups]
    offs = np.concatenate([[0], np.cumsum(rows)])
    machines = ",".join("127.0.0.1:%d" % (base_port + r) for r in range(R))
    out, errs = [None] * R, []

    def task(r):
        try:
            capi.set_device(r)
            capi.network_init(machines, base_port + r, 120, R)
            sl = slice(int(offs[r]), int(offs[r + 1]))
            ds = capi.Dataset.from_mat(X[sl], DS_PARAMS).set_field("label", y[sl])
            if weight is not None:
                ds.set_field("weight", weight[sl])
            if len(groups[r]) > 1 or groups[r][0] != rows[r]:
                ds.set_field("group", np.asarray(groups[r], np.int32))
            b = capi.Booster(ds, params)
            for _ in range(iters):
                fin = b.update_one_iter() if grad_fn is None else b.update_one_iter_custom(*grad_fn(r, b.get_scores()))
                if fin:
                    break
            out[r] = dict(model=b.save_model_to_string(), scores=b.get_scores())
            b.free()
            ds.free()
            capi.network_free()
        except Exception as e:   # noqa
            errs.append((r, repr(e)))

    ts = [threading.Thread(target=task, args=(r,)) for r in range(R)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(180)
    assert not errs, errs
    return out


def test_two_ranks_xendcg_seeds_each_ranks_queries_by_local_index(built):
    """Queries split at a group boundary; each rank's queries draw from LCGs seeded objective_seed + their rank-local index.  The built-in
    objective on two ranks equals the two-rank run fed the NumPy gradients of that seeding."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200.modeltext import compare_models, parse_model
    rng = np.random.default_rng(81)
    sizes = rng.integers(2, 40, 600).astype(np.int32)
    X, y = _rank_data(rng, sizes)
    groups = [sizes[:290], sizes[290:]]
    offs = [0, int(sizes[:290].sum())]
    params = _multi_params("rank_xendcg", 2, "objective_seed=7")
    rands = [R.xendcg_rands(len(g), 7) for g in groups]

    def grad(r, s):
        return R.xendcg_gradients(s, y[offs[r]:offs[r] + len(s)], groups[r], rands[r])[:2]

    built_in = _run_two_ranks(X, y, groups, params, 20, 24500)
    custom = _run_two_ranks(X, y, groups, params, 20, 24540, grad_fn=grad)
    assert built_in[1]["model"] == built_in[0]["model"]
    compare_models(parse_model(built_in[0]["model"]), parse_model(custom[0]["model"]))
    for r in range(2):
        np.testing.assert_allclose(built_in[r]["scores"], custom[r]["scores"], rtol=0, atol=1e-9)


def test_two_ranks_xentlambda_init_score_from_global_sums(built):
    """cross_entropy_lambda's init score on two ranks is log(expm1(global weighted label mean)), not a mean of the ranks' init scores"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200.modeltext import parse_model
    rng = np.random.default_rng(83)
    rows = [3000, 9000]
    n = sum(rows)
    X = rng.standard_normal((n, 4))
    y = np.concatenate([0.3 * rng.random(rows[0]), 0.5 + 0.5 * rng.random(rows[1])]).astype(np.float32)
    w = (0.5 + rng.random(n)).astype(np.float32)
    res = _run_two_ranks(X, y, [[rows[0]], [rows[1]]], _multi_params("cross_entropy_lambda", 2, "").replace("min_data_in_leaf=20", "min_data_in_leaf=1000000"),
                         1, 24580, weight=w)
    want = R.xentlambda_init_score(y, w)
    per_rank = np.mean([R.xentlambda_init_score(y[:rows[0]], w[:rows[0]]), R.xentlambda_init_score(y[rows[0]:], w[rows[0]:])])
    assert abs(want - per_rank) > 0.1
    for r in range(2):
        tree = parse_model(res[r]["model"])["trees"][0]
        assert tree["num_leaves"] == 1
        np.testing.assert_allclose(tree["leaf_value"], want, rtol=1e-12)
