"""Device evaluation of `average_precision` and `auc_mu` (with `auc_mu_weights`) through LGBM_BoosterGetEval, against scikit-learn and
brute-force NumPy restatements of the LightGBM 3.2 definitions.  Scores are set through init_score and evaluated before the first
iteration, at n = 300_001 rows, so that many blocks and a ragged tail occur; the training and validation sets are checked after a few
iterations too.  The early-stopping rule of the estimators ranks both names larger-is-better, which the last tests prove end to end."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 learning_rate=0.2 min_data_in_leaf=20 verbosity=-1 "
N = 300_001


def _booster(params, y, s, w=None):
    from mmlspark_b200 import capi
    X = np.random.default_rng(9).standard_normal((len(y), 2))
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y).set_field("init_score", np.ascontiguousarray(s, dtype=np.float64).ravel())
    if w is not None:
        ds.set_field("weight", w)
    try:
        return capi.Booster(ds, BASE + params), ds
    except Exception:
        ds.free()
        raise


def _eval_at_init(params, y, s, w=None):
    b, ds = _booster(params, y, s, w)
    try:
        return dict(zip(b.eval_names(), b.get_eval(0)))
    finally:
        b.free()
        ds.free()


def _weights(rng, n, zero_frac=0.05):
    """float32 weights in [0.5, 1.5) with some zeros: their double sums are exact, so the cub prefix sums are reproducible bit for bit"""
    w = (0.5 + rng.random(n)).astype(np.float32)
    w[rng.random(n) < zero_frac] = 0.0
    return w


def _aucmu_pairs(y, S, w):
    """the default-matrix reference: the mean over i < j of roc_auc_score(label == i, s_i - s_j) on the rows of classes i and j"""
    from sklearn.metrics import roc_auc_score
    K = S.shape[1]
    vals = []
    for i in range(K):
        for j in range(i + 1, K):
            m = (y == i) | (y == j)
            vals.append(roc_auc_score(y[m] == i, S[m, i] - S[m, j], sample_weight=None if w is None else w[m]))
    return float(np.mean(vals))


def _aucmu_brute(y, S, w, Wm):
    """O(n_i * n_j) restatement: d = t1 * sum_c v[c] s_c with v = Wm[i] - Wm[j], t1 = v[i] - v[j], diagonal of Wm zeroed"""
    K = S.shape[1]
    Wm = np.array(Wm, dtype=np.float64).reshape(K, K)
    np.fill_diagonal(Wm, 0.0)
    w = np.ones(len(y)) if w is None else w.astype(np.float64)
    tot = 0.0
    for i in range(K):
        for j in range(i + 1, K):
            v = Wm[i] - Wm[j]
            t1 = v[i] - v[j]
            dot = np.zeros(len(y))
            for c in range(K):
                if v[c] != 0.0:
                    dot = dot + v[c] * S[:, c]
            d = t1 * dot
            a, b = y == i, y == j
            da, db = d[a][:, None], d[b][None, :]
            wab = w[a][:, None] * w[b][None, :]
            num = (wab * ((da > db) + 0.5 * (da == db))).sum()
            tot += num / (w[a].sum() * w[b].sum())
    return 2.0 * tot / (K * (K - 1))


def _mc_scores(rng, y, K, decimals=None):
    """class-major [K][n] scores that favour the true class; rounded scores give exact ties"""
    n = len(y)
    S = rng.standard_normal((n, K)) + 1.2 * np.eye(K)[y.astype(int)]
    if decimals is not None:
        S = np.round(S, decimals)
    return S


# ------------------------------------------------------------------------------------------------ average_precision
@pytest.mark.parametrize("case", ["plain", "weighted", "coarse_ties", "signed_zeros"])
def test_average_precision_against_sklearn(built, case):
    from sklearn.metrics import average_precision_score
    rng = np.random.default_rng(100 + ["plain", "weighted", "coarse_ties", "signed_zeros"].index(case))
    y = (rng.random(N) < 0.2).astype(np.float32)
    s = rng.standard_normal(N) + 1.5 * y
    w = None
    if case == "weighted":
        w = _weights(rng, N)
    elif case == "coarse_ties":
        s = np.round(s, 0)                                     # a handful of values: large weighted tie groups
        w = _weights(rng, N)
        assert len(np.unique(s)) < 20
    elif case == "signed_zeros":
        s = np.array([0.0, -0.0, 1e-8, -1e-8, 0.5, -0.5])[rng.integers(0, 6, N)]
        w = _weights(rng, N)
    got = _eval_at_init("objective=binary metric=average_precision", y, s, w)["average_precision"]
    np.testing.assert_allclose(got, average_precision_score(y, s, sample_weight=w), rtol=1e-10)


def test_average_precision_signed_zeros_are_one_tie(built):
    """positives at +0.0 and negatives at -0.0 form one group: AP is the positive share"""
    y = (np.arange(N) % 3 == 0).astype(np.float32)
    s = np.where(y > 0, 0.0, -0.0)
    np.testing.assert_allclose(_eval_at_init("objective=binary metric=average_precision", y, s)["average_precision"], (y > 0).sum() / N, rtol=1e-14)


def test_average_precision_single_class_is_one(built):
    rng = np.random.default_rng(110)
    s = rng.standard_normal(N)
    w = _weights(rng, N)
    for label in (0.0, 1.0):
        assert _eval_at_init("objective=binary metric=average_precision", np.full(N, label, np.float32), s, w)["average_precision"] == 1.0


def test_average_precision_train_and_valid_after_iterations(built):
    from mmlspark_b200 import capi
    from sklearn.metrics import average_precision_score
    rng = np.random.default_rng(111)
    n, nv = N, 70_001
    X = np.round(rng.standard_normal((n + nv, 6)), 1)
    y = (X[:, 0] + 0.5 * X[:, 1] + 0.8 * rng.standard_normal(n + nv) > 1.0).astype(np.float32)
    w = _weights(rng, n + nv)
    ds = capi.Dataset.from_mat(X[:n], DS_PARAMS).set_field("label", y[:n]).set_field("weight", w[:n])
    dv = capi.Dataset.from_mat(X[n:], DS_PARAMS, reference=ds).set_field("label", y[n:]).set_field("weight", w[n:])
    b = capi.Booster(ds, BASE + "objective=binary metric=average_precision,auc")
    b.add_valid(dv)
    for _ in range(3):
        b.update_one_iter()
    assert b.eval_names() == ["average_precision", "auc"]
    for idx, sl in ((0, slice(0, n)), (1, slice(n, n + nv))):
        s = b.get_scores(idx)
        assert len(np.unique(s)) < len(s) / 4                # the tie groups really occur
        got = b.get_eval(idx)
        np.testing.assert_allclose(got[0], average_precision_score(y[sl], s, sample_weight=w[sl]), rtol=1e-10)
    b.free(); dv.free(); ds.free()


# ------------------------------------------------------------------------------------------------ auc_mu
@pytest.mark.parametrize("objective", ["multiclass", "multiclassova"])
@pytest.mark.parametrize("weighted", [False, True])
def test_auc_mu_default_matrix_against_sklearn(built, objective, weighted):
    """K = 5: the ten class pairs hold 4n items, more than the ~2n of one pair batch, so several batches run (K - 1 > 2).
    Scores rounded to one decimal give exact ties of s_i - s_j."""
    rng = np.random.default_rng(200 + weighted + 2 * (objective == "multiclassova"))
    K = 5
    y = rng.choice(K, N, p=[0.35, 0.3, 0.2, 0.1, 0.05]).astype(np.float32)
    S = _mc_scores(rng, y, K, decimals=1)
    w = _weights(rng, N) if weighted else None
    got = _eval_at_init("objective=%s num_class=%d metric=auc_mu" % (objective, K), y, S.T, w)["auc_mu"]
    np.testing.assert_allclose(got, _aucmu_pairs(y, S, w), rtol=1e-10)


def test_auc_mu_custom_matrix_against_brute_force(built):
    rng = np.random.default_rng(210)
    K, n = 4, 3001
    y = rng.integers(0, K, n).astype(np.float32)
    S = _mc_scores(rng, y, K)
    w = _weights(rng, n)
    Wm = rng.uniform(0.2, 3.0, (K, K))                         # dense and not symmetric
    np.fill_diagonal(Wm, 0.0)
    key = "auc_mu_weights=" + ",".join(repr(float(v)) for v in Wm.ravel())
    got = _eval_at_init("objective=multiclass num_class=%d metric=auc_mu %s" % (K, key), y, S.T, w)["auc_mu"]
    want = _aucmu_brute(y, S, w, Wm)
    np.testing.assert_allclose(got, want, rtol=1e-10)
    assert abs(want - _aucmu_brute(y, S, w, np.ones((K, K)))) > 1e-3      # the matrix matters
    # a non-zero diagonal is overwritten with 0
    Wd = Wm.copy()
    np.fill_diagonal(Wd, [5.0, -1.0, 2.0, 0.5])
    keyd = "auc_mu_weights=" + ",".join(repr(float(v)) for v in Wd.ravel())
    assert _eval_at_init("objective=multiclass num_class=%d metric=auc_mu %s" % (K, keyd), y, S.T, w)["auc_mu"] == got
    # the default matrix through the key equals no key
    ones = "auc_mu_weights=" + ",".join(["1"] * (K * K))
    a = _eval_at_init("objective=multiclass num_class=%d metric=auc_mu %s" % (K, ones), y, S.T, w)["auc_mu"]
    b = _eval_at_init("objective=multiclass num_class=%d metric=auc_mu" % K, y, S.T, w)["auc_mu"]
    assert a == b
    np.testing.assert_allclose(b, _aucmu_pairs(y, S, w), rtol=1e-10)


def test_auc_mu_absent_class_is_nan(built):
    """a class without rows in the evaluated set: its pairs divide 0 by 0 (upstream has no guard), so auc_mu is NaN"""
    rng = np.random.default_rng(220)
    K = 4
    y = rng.choice([0, 1, 3], N).astype(np.float32)
    S = _mc_scores(rng, y, K)
    assert np.isnan(_eval_at_init("objective=multiclass num_class=%d metric=auc_mu" % K, y, S.T)["auc_mu"])
    # a class whose rows all weigh 0 is absent by weight
    y = rng.integers(0, K, N).astype(np.float32)
    w = _weights(rng, N)
    w[y == 2] = 0.0
    S = _mc_scores(rng, y, K)
    assert np.isnan(_eval_at_init("objective=multiclass num_class=%d metric=auc_mu" % K, y, S.T, w)["auc_mu"])


# ------------------------------------------------------------------------------------------------ checks
def _small_ds(K, n=5000, seed=230, reference=None):
    from mmlspark_b200 import capi
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 4))
    y = rng.integers(0, K, n).astype(np.float32)
    return capi.Dataset.from_mat(X, DS_PARAMS, reference=reference).set_field("label", y), X, y


def test_auc_mu_needs_a_multiclass_objective(built):
    from mmlspark_b200 import capi
    ds, _, _ = _small_ds(2)
    with pytest.raises(capi.LightGBMError, match="needs a multiclass objective"):
        capi.Booster(ds, BASE + "objective=binary metric=auc_mu")
    ds.free()


def test_auc_mu_weights_length_checked_at_create_and_reset(built):
    from mmlspark_b200 import capi
    K = 3
    ds, _, _ = _small_ds(K)
    with pytest.raises(capi.LightGBMError, match="auc_mu_weights must have 9 elements"):
        capi.Booster(ds, BASE + "objective=multiclass num_class=3 metric=auc_mu auc_mu_weights=0,1,1,1,0,1,1,1")
    b = capi.Booster(ds, BASE + "objective=multiclass num_class=3 metric=multi_logloss,auc_mu")
    b.update_one_iter()
    before = b.get_eval(0)
    with pytest.raises(capi.LightGBMError, match="auc_mu_weights must have 9 elements"):
        b.reset_parameter("auc_mu_weights=1,2,3,4")
    after = b.get_eval(0)
    assert before.tobytes() == after.tobytes()
    assert "[auc_mu_weights: ]" in b.save_model_to_string()
    b.reset_parameter("auc_mu_weights=0,1,2,1,0,1,2,1,0")
    assert "[auc_mu_weights: 0,1,2,1,0,1,2,1,0]" in b.save_model_to_string()
    assert b.get_eval(0)[1] != before[1]
    b.free(); ds.free()


def test_auc_mu_validation_labels_checked(built):
    from mmlspark_b200 import capi
    K = 3
    ds, _, _ = _small_ds(K)
    b = capi.Booster(ds, BASE + "objective=multiclass num_class=3 metric=auc_mu")
    dv, _, _ = _small_ds(K, n=2000, seed=231, reference=ds)
    yv = np.random.default_rng(232).integers(0, K, 2000).astype(np.float32)
    yv[77] = 3.0
    dv.set_field("label", yv)
    with pytest.raises(capi.LightGBMError, match=r"Label must be in \[0, 3\)"):
        b.add_valid(dv)
    yv[77] = -1.0
    dv.set_field("label", yv)
    with pytest.raises(capi.LightGBMError, match=r"Label must be in \[0, 3\)"):
        b.add_valid(dv)
    yv[77] = 2.0
    dv.set_field("label", yv)
    b.add_valid(dv)
    assert np.isfinite(b.get_eval(1)).all()
    b.free(); dv.free(); ds.free()


def test_auc_mu_names_order_and_other_metrics_unchanged(built):
    rng = np.random.default_rng(240)
    K = 4
    y = rng.integers(0, K, N).astype(np.float32)
    S = _mc_scores(rng, y, K, decimals=2)
    w = _weights(rng, N)
    b, ds = _booster("objective=multiclass num_class=%d metric=multi_logloss,auc_mu,multi_error" % K, y, S.T, w)
    b0, ds0 = _booster("objective=multiclass num_class=%d metric=multi_logloss,multi_error" % K, y, S.T, w)
    try:
        assert b.eval_names() == ["multi_logloss", "auc_mu", "multi_error"]
        for _ in range(2):
            b.update_one_iter()
            b0.update_one_iter()
        got, ref = b.get_eval(0), b0.get_eval(0)
        assert got[0].tobytes() == ref[0].tobytes() and got[2].tobytes() == ref[1].tobytes()
        np.testing.assert_allclose(got[1], _aucmu_pairs(y, b.get_scores(0).reshape(K, N).T, w), rtol=1e-10)
    finally:
        b.free(); ds.free(); b0.free(); ds0.free()


def test_repeated_evaluations_are_bit_identical(built):
    rng = np.random.default_rng(250)
    K = 5
    y = rng.integers(0, K, N).astype(np.float32)
    S = _mc_scores(rng, y, K)
    w = _weights(rng, N)
    b, ds = _booster("objective=multiclass num_class=%d metric=auc_mu" % K, y, S.T, w)
    try:
        assert b.get_eval(0).tobytes() == b.get_eval(0).tobytes()
    finally:
        b.free(); ds.free()
    yb = (y > 2).astype(np.float32)
    b, ds = _booster("objective=binary metric=average_precision,auc", yb, S[:, 0], w)
    try:
        assert b.get_eval(0).tobytes() == b.get_eval(0).tobytes()
    finally:
        b.free(); ds.free()


# ------------------------------------------------------------------------------------------------ two ranks on one device
def test_two_ranks_on_one_device_are_rank_local(built):
    """data-parallel with both ranks on device 0 (the same-device collective): each rank reports average_precision and auc_mu on its
    own shard, nothing is all-reduced"""
    import test_gpu_multi as M
    from tree_check import on_ranks
    from mmlspark_b200 import capi
    from sklearn.metrics import average_precision_score
    rng = np.random.default_rng(260)
    n, K = 60_000, 3
    X = rng.standard_normal((n, 8))
    yc = np.argmax(X[:, :K] + 0.7 * rng.standard_normal((n, K)), axis=1).astype(np.float32)
    yb = (yc == 0).astype(np.float32)
    rank_rows = [n // 2 + 1234, n - n // 2 - 1234]
    offs = np.concatenate([[0], np.cumsum(rank_rows)])

    def body(r):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        out = {}
        for name, y, extra in (("ap", yb, "metric=average_precision"), ("mu", yc, "num_class=%d metric=auc_mu" % K)):
            objective = "binary" if name == "ap" else "multiclass"
            ds = capi.Dataset.from_mat(X[sl], M.DS_PARAMS).set_field("label", y[sl])
            b = capi.Booster(ds, M._params(objective, 2, extra))
            for _ in range(3):
                b.update_one_iter()
            out[name] = (b.get_eval(0)[0], b.get_scores(0))
            b.free(); ds.free()
        return out

    res, errs = on_ranks(2, 26800, body)
    assert not errs, errs
    for r in range(2):
        sl = slice(int(offs[r]), int(offs[r + 1]))
        ap, s = res[r]["ap"]
        np.testing.assert_allclose(ap, average_precision_score(yb[sl], s), rtol=1e-10)
        mu, s = res[r]["mu"]
        np.testing.assert_allclose(mu, _aucmu_pairs(yc[sl], s.reshape(K, -1).T, None), rtol=1e-10)
    assert res[0]["ap"][0] != res[1]["ap"][0]


# ------------------------------------------------------------------------------------------------ estimators
def _collecting_delegate():
    from mmlspark_b200.lightgbm import LightGBMDelegate

    class D(LightGBMDelegate):
        def __init__(self):
            self.valid = []

        def afterTrainIteration(self, batchIndex, partitionId, curIters, trainParams, booster, hasValid, isFinished, trainEvalResults,
                                validEvalResults):
            if validEvalResults is not None:
                self.valid.append((curIters, dict(validEvalResults)))
    return D()


@pytest.mark.parametrize("kind", ["multiclass_auc_mu", "binary_average_precision"])
def test_estimator_early_stops_larger_is_better(built, kind):
    from mmlspark_b200.lightgbm import Frame, LightGBMClassifier
    rng = np.random.default_rng(270)
    n, F = 12000, 10
    X = rng.standard_normal((n, F))
    if kind == "multiclass_auc_mu":
        y = np.argmax(X[:, :3] + 1.0 * rng.standard_normal((n, 3)), axis=1).astype(np.float64)
        metric, extra = "auc_mu", dict(objective="multiclass")
    else:
        s = X[:, 0] + 0.8 * X[:, 1] * X[:, 2] + 0.9 * rng.standard_normal(n)
        y = (s > np.quantile(s, 0.9)).astype(np.float64)      # imbalanced
        metric, extra = "average_precision", {}
    df = Frame({"features": X, "label": y}).with_column("valid", rng.random(n) < 0.3)
    d = _collecting_delegate()
    m = LightGBMClassifier(numIterations=300, numTasks=1, learningRate=0.3, numLeaves=63, validationIndicatorCol="valid",
                           earlyStoppingRound=5, metric=metric, delegate=d, **extra).fit(df)
    assert 0 < m.getBoosterNumTotalIterations() < 300
    iters = [it for it, _ in d.valid]
    vals = np.array([v[metric] for _, v in d.valid])
    assert iters == list(range(len(iters))) and np.isfinite(vals).all()
    assert m.getBoosterBestIteration() == iters[int(np.argmax(vals))]
    assert np.argmax(vals) != np.argmin(vals)                  # the rule told the two directions apart
