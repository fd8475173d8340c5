"""Device-side evaluation (LGBM_BoosterGetEval; TrainUtils.scala:125-151 drives early stopping with it) against independent numpy /
scikit-learn restatements of the LightGBM metric definitions, on the training scores (data_idx 0) and a validation set (data_idx 1)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 learning_rate=0.2 min_data_in_leaf=20 verbosity=-1 "


def _fit(X, y, params, Xv=None, yv=None, weight=None, wv=None, group=None, gv=None, iters=5):
    from mmlspark_b200 import capi
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    if weight is not None:
        ds.set_field("weight", weight)
    if group is not None:
        ds.set_field("group", group)
    b = capi.Booster(ds, BASE + params)
    dv = None
    if Xv is not None:
        dv = capi.Dataset.from_mat(Xv, DS_PARAMS, reference=ds).set_field("label", yv)
        if wv is not None:
            dv.set_field("weight", wv)
        if gv is not None:
            dv.set_field("group", gv)
        b.add_valid(dv)
    for _ in range(iters):
        b.update_one_iter()
    return b, ds, dv


def _wavg(loss, w):
    w = np.ones_like(loss) if w is None else w.astype(np.float64)
    return float((loss * w).sum() / w.sum())


def test_binary_metrics_incl_weighted_auc_with_ties(built):
    from sklearn.metrics import roc_auc_score
    rng = np.random.default_rng(1)
    n = 30000
    X = np.round(rng.standard_normal((n, 6)), 1)            # coarse features => many tied scores
    y = (X[:, 0] + 0.5 * X[:, 1] + 0.8 * rng.standard_normal(n) > 0).astype(np.float32)
    w = (0.5 + rng.random(n)).astype(np.float32)
    Xv, yv, wv = X[:7000] + 0.1, y[:7000], w[:7000]
    b, _, _ = _fit(X, y, "objective=binary metric=auc,binary_logloss,binary_error", Xv, yv, w, wv, iters=3)
    assert b.eval_names() == ["auc", "binary_logloss", "binary_error"]
    for idx, (yy, ww) in enumerate(((y, w), (yv, wv))):
        s = b.get_scores(idx)
        p = 1.0 / (1.0 + np.exp(-s))
        got = b.get_eval(idx)
        assert len(np.unique(s)) < len(s) / 4                # the tie groups really occur
        np.testing.assert_allclose(got[0], roc_auc_score(yy, s, sample_weight=ww), rtol=1e-10)
        pl = np.where(yy > 0, p, 1 - p)
        np.testing.assert_allclose(got[1], _wavg(-np.log(np.maximum(pl, 1e-15)), ww), rtol=1e-12)
        np.testing.assert_allclose(got[2], _wavg(((p <= 0.5) == (yy > 0)).astype(np.float64), ww), rtol=1e-12)


def test_regression_metrics(built):
    rng = np.random.default_rng(2)
    n = 20000
    X = rng.standard_normal((n, 5))
    y = (np.exp(0.3 * X[:, 0]) + 0.1 * np.abs(rng.standard_normal(n))).astype(np.float32)
    w = (0.5 + rng.random(n)).astype(np.float32)
    names = "l2,rmse,l1,huber,fair,quantile,mape,poisson,tweedie"
    b, _, _ = _fit(X, y, "objective=regression alpha=0.7 fair_c=1.3 tweedie_variance_power=1.4 metric=" + names, weight=w)
    s = b.get_scores(0)
    got = dict(zip(b.eval_names(), b.get_eval(0)))
    d = s - y
    want = {
        "l2": _wavg(d * d, w), "rmse": np.sqrt(_wavg(d * d, w)), "l1": _wavg(np.abs(d), w),
        "huber": _wavg(np.where(np.abs(d) <= 0.7, 0.5 * d * d, 0.7 * (np.abs(d) - 0.35)), w),
        "fair": _wavg(1.3 * np.abs(d) - 1.69 * np.log(1 + np.abs(d) / 1.3), w),
        "quantile": _wavg(np.where(y - s < 0, (0.7 - 1) * (y - s), 0.7 * (y - s)), w),
        "mape": _wavg(np.abs(y - s) / np.maximum(1.0, np.abs(y)), w),
        "poisson": _wavg(np.maximum(np.exp(s), 1e-10) - y * np.log(np.maximum(np.exp(s), 1e-10)), w),
        "tweedie": _wavg(-y * np.exp((1 - 1.4) * np.log(np.maximum(np.exp(s), 1e-10))) / (1 - 1.4) + np.exp((2 - 1.4) * np.log(np.maximum(np.exp(s), 1e-10))) / (2 - 1.4), w),
    }
    for k, v in want.items():
        np.testing.assert_allclose(got[k], v, rtol=1e-11, err_msg=k)


@pytest.mark.parametrize("objective", ["multiclass", "multiclassova"])
def test_multiclass_metrics(built, objective):
    rng = np.random.default_rng(3)
    n, K = 20000, 4
    X = rng.standard_normal((n, 6))
    y = np.argmax(X[:, :K] + 0.7 * rng.standard_normal((n, K)), axis=1).astype(np.float32)
    b, _, _ = _fit(X, y, "objective=%s num_class=4 metric=multi_logloss,multi_error" % objective)
    s = b.get_scores(0).reshape(K, n).T
    if objective == "multiclass":
        e = np.exp(s - s.max(axis=1, keepdims=True))
        p = e / e.sum(axis=1, keepdims=True)
    else:
        p = 1.0 / (1.0 + np.exp(-s))
    pl = p[np.arange(n), y.astype(int)]
    got = b.get_eval(0)
    np.testing.assert_allclose(got[0], np.mean(-np.log(np.maximum(pl, 1e-15))), rtol=1e-12)
    np.testing.assert_allclose(got[1], np.mean((p >= pl[:, None]).sum(axis=1) > 1), rtol=1e-12)


def _rank_metrics(s, y, sizes, ks, gain):
    nd, mp = np.zeros(len(ks)), np.zeros(len(ks))
    off = 0
    for c in sizes:
        ss, yy = s[off:off + c], y[off:off + c].astype(int)
        off += c
        order = np.argsort(-ss, kind="stable")
        ideal = np.sort(yy)[::-1]
        npos = int((yy > 0.5).sum())
        for e, k in enumerate(ks):
            kk = min(k, c)
            disc = 1.0 / np.log2(2.0 + np.arange(kk))
            maxdcg = float((gain[ideal[:kk]] * disc).sum())
            nd[e] += 1.0 if maxdcg <= 0 else float((gain[yy[order[:kk]]] * disc).sum()) / maxdcg
            hits = (yy[order[:kk]] > 0.5)
            ap = float((np.cumsum(hits)[hits] / (np.nonzero(hits)[0] + 1.0)).sum())
            mp[e] += ap / min(npos, kk) if npos > 0 else 1.0
    return nd / len(sizes), mp / len(sizes)


def test_ranking_metrics_ndcg_and_map(built):
    rng = np.random.default_rng(4)
    sizes = rng.integers(1, 60, 800).astype(np.int32)
    sizes[5] = 300                                          # one query longer than the block
    n = int(sizes.sum())
    X = np.round(rng.standard_normal((n, 5)), 1)
    y = np.clip(np.round(X[:, 0] + 0.7 * rng.standard_normal(n) + 1.0), 0, 4).astype(np.float32)
    y[:sizes[0]] = 0                                        # an all-irrelevant query: ndcg = map = 1 by definition
    ks = [1, 3, 5, 10]
    # validation set = a prefix made of whole queries
    cut = int(np.searchsorted(np.cumsum(sizes), n // 2, side="right"))
    from mmlspark_b200 import capi
    nv = int(sizes[:cut].sum())
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y).set_field("group", sizes)
    dv = capi.Dataset.from_mat(X[:nv], DS_PARAMS, reference=ds).set_field("label", y[:nv]).set_field("group", sizes[:cut])
    b = capi.Booster(ds, BASE + "objective=lambdarank metric=ndcg,map eval_at=1,3,5,10 min_data_in_leaf=5")
    b.add_valid(dv)
    for _ in range(4):
        b.update_one_iter()
    assert b.eval_names() == ["ndcg@1", "ndcg@3", "ndcg@5", "ndcg@10", "map@1", "map@3", "map@5", "map@10"]
    gain = np.array([0.0] + [float((1 << i) - 1) for i in range(1, 31)])
    for idx, (nn, sz) in enumerate(((n, sizes), (nv, sizes[:cut]))):
        s = b.get_scores(idx)
        nd, mp = _rank_metrics(s, y[:nn], sz, ks, gain)
        got = b.get_eval(idx)
        np.testing.assert_allclose(got[:4], nd, rtol=1e-10)
        np.testing.assert_allclose(got[4:], mp, rtol=1e-6)          # [UPSTREAM] accumulates num_hit / (j + 1.0f) in float


# ------------------------------------------------------------------------------------------------ metrics at chosen scores
# get_eval before the first iteration evaluates the init scores exactly, so the scores can sit where each metric clips.
N_EDGE = 300_001        # the metric kernels' blocks take contiguous row ranges; this n spans many of them and ends on a ragged tail
EDGE_SCORES = np.array([0.0, -0.0, 1e-8, -1e-8, 0.5, -0.5, 5.0, -5.0, 23.0, -23.0, 23.1, -23.1, 30.0, -30.0, 37.0, -37.0, 40.0, -40.0])


def _edge_scores(rng, n, spread=3.0):
    s = spread * rng.standard_normal(n)
    pick = rng.random(n) < 0.5
    s[pick] = EDGE_SCORES[rng.integers(0, len(EDGE_SCORES), int(pick.sum()))]
    return s


def _eval_at_init(params, y, s, w=None):
    from mmlspark_b200 import capi
    X = np.random.default_rng(9).standard_normal((len(y), 2))
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y).set_field("init_score", s)
    if w is not None:
        ds.set_field("weight", w)
    b = capi.Booster(ds, BASE + params)
    try:
        return dict(zip(b.eval_names(), b.get_eval(0)))
    finally:
        b.free()
        ds.free()


def _safe_log(x):
    return np.where(x > 0, np.log(np.where(x > 0, x, 1.0)), -np.inf)


@pytest.mark.parametrize("weighted", [False, True])
def test_regression_metrics_at_clipping_scores(built, weighted):
    """poisson and tweedie clip exp(score) at 1e-10 (score <= -23.03); the exp-link metrics are evaluated with their objectives."""
    rng = np.random.default_rng(10 + weighted)
    n = N_EDGE
    y = (0.1 + rng.gamma(2.0, 1.5, n)).astype(np.float32)          # > 0: gamma's log(label)
    s = _edge_scores(rng, n)
    w = (0.5 + rng.random(n)).astype(np.float32) if weighted else None
    y64 = y.astype(np.float64)
    with np.errstate(all="ignore"):
        d = s - y64
        got = _eval_at_init("objective=regression alpha=0.7 fair_c=1.3 metric=l2,rmse,l1,huber,fair,quantile,mape", y, s, w)
        want = {
            "l2": _wavg(d * d, w), "rmse": np.sqrt(_wavg(d * d, w)), "l1": _wavg(np.abs(d), w),
            "huber": _wavg(np.where(np.abs(d) <= 0.7, 0.5 * d * d, 0.7 * (np.abs(d) - 0.35)), w),
            "fair": _wavg(1.3 * np.abs(d) - 1.69 * np.log(1 + np.abs(d) / 1.3), w),
            "quantile": _wavg(np.where(y64 - s < 0, (0.7 - 1) * (y64 - s), 0.7 * (y64 - s)), w),
            "mape": _wavg(np.abs(y64 - s) / np.maximum(1.0, np.abs(y64)), w),
        }
        sc = np.maximum(np.exp(s), 1e-10)
        got.update(_eval_at_init("objective=poisson metric=poisson", y, s, w))
        want["poisson"] = _wavg(sc - y64 * np.log(sc), w)
        got.update(_eval_at_init("objective=tweedie tweedie_variance_power=1.4 metric=tweedie", y, s, w))
        want["tweedie"] = _wavg(-y64 * np.exp((1 - 1.4) * np.log(sc)) / (1 - 1.4) + np.exp((2 - 1.4) * np.log(sc)) / (2 - 1.4), w)
        got.update(_eval_at_init("objective=gamma metric=gamma,gamma_deviance", y, s, w))
        e = np.exp(s)
        theta = -1.0 / e
        want["gamma"] = _wavg(-((y64 * theta + _safe_log(-theta)) + (_safe_log(y64) - _safe_log(y64))), w)
        tmp = y64 / (e + 1e-9)
        want["gamma_deviance"] = _wavg(tmp - _safe_log(tmp) - 1, w)
    assert (s <= -23.1).any() and sorted(got) == sorted(want)
    for k, v in want.items():
        np.testing.assert_allclose(got[k], v, rtol=1e-11, err_msg=k)


@pytest.mark.parametrize("sigmoid", [1.0, 2.0])
def test_binary_and_xentropy_metrics_at_saturating_scores(built, sigmoid):
    """|sigmoid * score| >= 37 rounds p to 1 in fp64: logloss takes its epsilon branch, cross_entropy its 1e-12 branch."""
    rng = np.random.default_rng(20 + int(sigmoid))
    n = N_EDGE
    s = _edge_scores(rng, n, spread=20.0)
    y = (rng.random(n) < 0.3).astype(np.float32)
    w = (0.5 + rng.random(n)).astype(np.float32)
    w[rng.random(n) < 0.05] = 0.0
    got = _eval_at_init("objective=binary sigmoid=%g metric=binary_logloss,binary_error" % sigmoid, y, s, w)
    p = 1.0 / (1.0 + np.exp(-sigmoid * s))
    pl = np.where(y > 0, p, 1.0 - p)
    assert (pl == 0).any()
    np.testing.assert_allclose(got["binary_logloss"], _wavg(np.where(pl > 1e-15, -np.log(np.maximum(pl, 1e-300)), -np.log(1e-15)), w), rtol=1e-12)
    np.testing.assert_allclose(got["binary_error"], _wavg(((p <= 0.5) == (y > 0)).astype(np.float64), w), rtol=1e-12)
    yx = np.where(rng.random(n) < 0.5, y, rng.random(n)).astype(np.float32)      # probabilities: 0, 1 and fractions
    got = _eval_at_init("objective=cross_entropy metric=cross_entropy", yx, s, w)
    y64 = yx.astype(np.float64)
    with np.errstate(all="ignore"):
        p = 1.0 / (1.0 + np.exp(-s))
        a = y64 * np.where(p > 1e-12, np.log(np.maximum(p, 1e-300)), np.log(1e-12))
        b = (1.0 - y64) * np.where(1.0 - p > 1e-12, np.log(np.maximum(1.0 - p, 1e-300)), np.log(1e-12))
    np.testing.assert_allclose(got["cross_entropy"], _wavg(-(a + b), w), rtol=1e-12)


@pytest.mark.parametrize("objective", ["multiclass", "multiclassova"])
def test_multiclass_metrics_at_extreme_scores(built, objective):
    rng = np.random.default_rng(30)
    n, K = N_EDGE, 5
    y = rng.integers(0, K, n).astype(np.float32)
    s = np.concatenate([_edge_scores(rng, n, spread=10.0) for _ in range(K)])
    got = _eval_at_init("objective=%s num_class=%d metric=multi_logloss,multi_error" % (objective, K), y, s)
    sk = s.reshape(K, n).T
    if objective == "multiclass":
        e = np.exp(sk - sk.max(axis=1, keepdims=True))
        p = e / e.sum(axis=1, keepdims=True)
    else:
        p = 1.0 / (1.0 + np.exp(-sk))
    pl = p[np.arange(n), y.astype(int)]
    assert (pl <= 1e-15).any()
    np.testing.assert_allclose(got["multi_logloss"], np.mean(np.where(pl > 1e-15, -np.log(np.maximum(pl, 1e-300)), -np.log(1e-15))), rtol=1e-12)
    np.testing.assert_allclose(got["multi_error"], np.mean((p >= pl[:, None]).sum(axis=1) > 1), rtol=1e-12)


def test_auc_treats_signed_zeros_as_one_tie(built):
    """-0.0 == +0.0, so they form one tie group, as in LightGBM's `cur_score != threshold` and in sklearn; a user init_score can hold -0.0."""
    from sklearn.metrics import roc_auc_score
    n = N_EDGE
    y = (np.arange(n) % 3 == 0).astype(np.float32)
    s = np.where(y > 0, 0.0, -0.0)             # positives at +0.0, negatives at -0.0: one tie, AUC 1/2
    assert _eval_at_init("objective=binary metric=auc", y, s)["auc"] == 0.5
    rng = np.random.default_rng(40)
    y = (rng.random(n) < 0.4).astype(np.float32)
    s = np.array([0.0, -0.0, 1e-8, -1e-8, 0.5, -0.5])[rng.integers(0, 6, n)]
    w = (0.5 + rng.random(n)).astype(np.float32)
    got = _eval_at_init("objective=binary metric=auc", y, s, w)["auc"]
    np.testing.assert_allclose(got, roc_auc_score(y, s, sample_weight=w), rtol=1e-10)


def test_auc_weighted_ties_and_single_class(built):
    from sklearn.metrics import roc_auc_score
    rng = np.random.default_rng(41)
    n = N_EDGE
    s = np.round(_edge_scores(rng, n), 0)       # few distinct values: large weighted tie groups
    y = (rng.random(n) < 1.0 / (1.0 + np.exp(-np.clip(s, -30, 30)))).astype(np.float32)
    w = (10.0 ** rng.uniform(-3, 3, n)).astype(np.float32)
    w[rng.random(n) < 0.05] = 0.0
    got = _eval_at_init("objective=binary metric=auc", y, s, w)["auc"]
    np.testing.assert_allclose(got, roc_auc_score(y, s, sample_weight=w), rtol=1e-10)
    for label in (0.0, 1.0):                    # one class only: LightGBM reports 1
        assert _eval_at_init("objective=binary metric=auc", np.full(n, label, np.float32), s, w)["auc"] == 1.0


def test_unknown_metric_fails_at_booster_create(built):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(5)
    X = rng.standard_normal((2000, 4))
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", X[:, 0].astype(np.float32))
    with pytest.raises(capi.LightGBMError):
        capi.Booster(ds, BASE + "objective=regression metric=l2,not_a_metric")


def _error_data(n=2000, seed=6):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 4))
    return X, (X[:, 0] > 0).astype(np.float32)


def test_metric_errors_are_raised_by_the_call_that_meets_them(built):
    """Each metric error at the call that raises it: LGBM_BoosterCreate and LGBM_BoosterResetParameter reject the metric list, GetEval
    what it finds in the data it evaluates; a rejected reset leaves the names and values of every evaluation as they were."""
    from mmlspark_b200 import capi
    X, y = _error_data()
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    many = "eval_at=" + ",".join(str(k) for k in range(1, 18))
    for params, match in (("objective=regression metric=l2,not_a_metric", "Unknown metric type name: not_a_metric"),
                          ("objective=regression metric=ndcg " + many, "eval_at: at most 16 positions are supported"),
                          ("objective=multiclass num_class=2 metric=kldiv", "metric kullback_leibler needs a single-output objective")):
        with pytest.raises(capi.LightGBMError, match=match):
            capi.Booster(ds, BASE + params)

    # create succeeds; the evaluation fails
    b, _, _ = _fit(X, y, "objective=binary metric=multi_logloss", X[:500], y[:500], iters=1)
    for idx in (0, 1):
        with pytest.raises(capi.LightGBMError, match="metric multi_logloss needs a multiclass objective"):
            b.get_eval(idx)
    for metric, name in (("ndcg", "NDCG"), ("map", "MAP")):
        b, _, _ = _fit(X, y, "objective=regression metric=" + metric, X[:500], y[:500], iters=1)
        assert b.eval_names() == [metric + "@%d" % k for k in range(1, 6)]
        for idx in (0, 1):
            with pytest.raises(capi.LightGBMError, match="The %s metric requires query information" % name):
                b.get_eval(idx)
    Xb, yb = _error_data(13_000, seed=7)      # one query of 13000 documents: more shared memory than the rank kernel may take
    b, _, _ = _fit(Xb, yb, "objective=regression metric=map", group=np.array([13_000], np.int32), iters=1)
    with pytest.raises(capi.LightGBMError, match="a query group is too large for the ranking metric kernel"):
        b.get_eval(0)

    # resets that fail every check of create and of the validation data
    b, _, _ = _fit(X, y, "objective=binary metric=binary_logloss,auc,l2", X[:500], y[:500], iters=2)
    names, evals = b.eval_names(), [b.get_eval(idx).tobytes() for idx in (0, 1)]
    yv_bad = y[:500].copy()
    yv_bad[3] = 2.0
    b2, _, _ = _fit(X, y, "objective=binary metric=binary_logloss", X[:500], yv_bad, iters=2)
    names2, evals2 = b2.eval_names(), [b2.get_eval(idx).tobytes() for idx in (0, 1)]
    for booster, params, match in ((b, "metric=l2,auc,bogus_metric", "Unknown metric type name: bogus_metric"),
                                   (b, "metric=ndcg " + many, "eval_at: at most 16 positions are supported"),
                                   (b, "metric=auc_mu", "metric auc_mu needs a multiclass objective"),
                                   (b2, "metric=binary_logloss,cross_entropy_lambda", r"\[cross_entropy_lambda\]: does not tolerate label 2")):
        with pytest.raises(capi.LightGBMError, match=match):
            booster.reset_parameter(params)
    assert b.eval_names() == names and [b.get_eval(idx).tobytes() for idx in (0, 1)] == evals
    assert b2.eval_names() == names2 and [b2.get_eval(idx).tobytes() for idx in (0, 1)] == evals2


def test_data_idx_out_of_range_is_rejected(built):
    """GetEval, GetNumPredict, GetPredict and the raw scores accept data_idx 0 (training) up to the number of validation sets"""
    import ctypes as C
    from mmlspark_b200 import capi
    X, y = _error_data()
    b, _, _ = _fit(X, y, "objective=binary metric=binary_logloss,auc", X[:500], y[:500], iters=2)
    before = [(b.get_eval(idx).tobytes(), b.get_predict(idx).tobytes(), b.get_scores(idx).tobytes()) for idx in (0, 1)]
    L, out, n = capi.load(), np.zeros(len(X), np.float64), C.c_int64(0)
    for idx in (-1, 2):
        # get_predict / get_scores call GetNumPredict first, so GetPredict and GetScores are also called on their own
        for call in (b.get_eval, b.get_predict, b.get_scores,
                     lambda i: capi.check(L.LGBM_BoosterGetPredict(b.handle, C.c_int(i), C.byref(n), capi._ptr(out))),
                     lambda i: capi.check(L.B200GBM_BoosterGetScores(b.handle, C.c_int(i), capi._ptr(out)))):
            with pytest.raises(capi.LightGBMError, match="data_idx out of range"):
                call(idx)
    assert not out.any()
    assert [(b.get_eval(idx).tobytes(), b.get_predict(idx).tobytes(), b.get_scores(idx).tobytes()) for idx in (0, 1)] == before


def test_booster_from_model_string_has_no_metrics(built):
    """A booster loaded from a model string evaluates nothing, so it lists no metric names, also after a parameter reset (LightGBM's
    GetEvalCounts of a loaded model is 0)"""
    from mmlspark_b200 import capi
    X, y = _error_data()
    b, _, _ = _fit(X, y, "objective=binary metric=binary_logloss,auc", iters=2)
    loaded = capi.Booster(model_str=b.save_model_to_string())
    assert loaded.eval_names() == []
    loaded.reset_parameter("metric=auc,l2")
    assert loaded.eval_names() == []
    with pytest.raises(capi.LightGBMError, match="loaded from a model string"):
        loaded.get_eval(0)
