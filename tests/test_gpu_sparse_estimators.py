"""The estimators on a scipy.sparse features column: fitted through LGBM_DatasetCreateFromCSR they give the native model the dense column
gives, under every matrixType, and transform() through the batched CSR predictor gives every column the dense input gives, bit for bit,
and what the per-row CSR predictor gives (SHAP values to 1e-12, as for dense rows).  Also: a bundled one-hot fit, validation with early
stopping, numBatches, two tasks, and a 2^18-column fit and transform that never builds a dense matrix."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu


def _ngpu():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout.count("GPU ")
    except Exception:
        return 0


def _data(seed, n=4000, F=30):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, F))
    X[rng.random((n, F)) < 0.7] = 0.0
    X[rng.random((n, F)) < 0.03] = np.nan
    z = np.nan_to_num(X[:, 0]) * 2 - np.nan_to_num(X[:, 1]) + np.nan_to_num(X[:, 2]) * np.nan_to_num(X[:, 3]) + 0.3 * rng.standard_normal(n)
    return rng, X, z


def _frame(X, cols):
    from mmlspark_b200.lightgbm import Frame
    return Frame(dict(cols, features=X))


def _model_string(m):
    return m.getNativeModel()


def _check_transform(m, Xd, cols, row_fns):
    """every column of transform() on sparse rows equals the dense rows' and the per-row CSR predictor's"""
    Xs = sp.csr_matrix(Xd)
    ts = m.transform(_frame(Xs, {}))
    td = m.transform(_frame(Xd, {}))
    for c in cols:
        np.testing.assert_array_equal(ts[c], td[c], err_msg=c)
    for r in np.random.default_rng(0).choice(Xd.shape[0], 25, replace=False):
        for c, fn in row_fns.items():
            if c == "shap":          # host TreeSHAP vs the device kernel: to 1e-12, as for dense rows (test_gpu_parity.py)
                np.testing.assert_allclose(fn(Xs[r]), ts[c][r], rtol=0, atol=1e-12, err_msg=c)
            else:
                np.testing.assert_array_equal(np.asarray(fn(Xs[r])), ts[c][r], err_msg=c)


def test_classifier_sparse_fit_and_transform(built):
    from mmlspark_b200.lightgbm import LightGBMClassifier
    _, X, z = _data(1)
    y = (z > np.median(z)).astype(np.float64)
    kw = dict(numIterations=12, numTasks=1, minDataInLeaf=5, leafPredictionCol="leaf", featuresShapCol="shap")
    md = LightGBMClassifier(**kw).fit(_frame(X, {"label": y}))
    ms = LightGBMClassifier(**kw).fit(_frame(sp.csr_matrix(X), {"label": y}))
    assert _model_string(ms) == _model_string(md)
    assert _model_string(LightGBMClassifier(matrixType="dense", **kw).fit(_frame(sp.csr_matrix(X), {"label": y}))) == _model_string(md)
    assert _model_string(LightGBMClassifier(matrixType="sparse", **kw).fit(_frame(X, {"label": y}))) == _model_string(md)
    b = ms.booster
    _check_transform(ms, X, ["rawPrediction", "probability", "prediction", "leaf", "shap"],
                     {"rawPrediction": lambda r: b.score(r, True, True), "probability": lambda r: b.score(r, False, True),
                      "leaf": b.predictLeaf, "shap": b.featuresShap})


def test_multiclass_classifier_sparse(built):
    from mmlspark_b200.lightgbm import LightGBMClassifier
    _, X, z = _data(2)
    y = np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])).astype(np.float64)
    kw = dict(objective="multiclass", numIterations=8, numTasks=1, minDataInLeaf=5, featuresShapCol="shap")
    md = LightGBMClassifier(**kw).fit(_frame(X, {"label": y}))
    ms = LightGBMClassifier(**kw).fit(_frame(sp.csr_matrix(X), {"label": y}))
    assert _model_string(ms) == _model_string(md)
    b = ms.booster
    _check_transform(ms, X, ["rawPrediction", "probability", "prediction", "shap"],
                     {"probability": lambda r: b.score(r, False, True), "shap": b.featuresShap})


def test_regressor_sparse_fit_and_transform(built):
    from mmlspark_b200.lightgbm import LightGBMRegressor
    _, X, z = _data(3)
    kw = dict(numIterations=12, numTasks=1, minDataInLeaf=5, leafPredictionCol="leaf", featuresShapCol="shap")
    md = LightGBMRegressor(**kw).fit(_frame(X, {"label": z}))
    ms = LightGBMRegressor(**kw).fit(_frame(sp.csr_matrix(X), {"label": z}))
    assert _model_string(ms) == _model_string(md)
    assert _model_string(LightGBMRegressor(matrixType="dense", **kw).fit(_frame(sp.csr_matrix(X), {"label": z}))) == _model_string(md)
    assert _model_string(LightGBMRegressor(matrixType="sparse", **kw).fit(_frame(X, {"label": z}))) == _model_string(md)
    b = ms.booster
    _check_transform(ms, X, ["prediction", "leaf", "shap"], {"prediction": ms.predict, "leaf": b.predictLeaf, "shap": b.featuresShap})
    r = sp.csr_matrix(X[:1])
    assert ms.getFeatureShaps(r) == md.getFeatureShaps(X[0])


def test_ranker_sparse_fit_and_transform(built):
    from mmlspark_b200.lightgbm import LightGBMRanker
    rng, X, z = _data(4)
    q = np.repeat(np.arange(200), 20)
    rng.shuffle(q)
    rel = np.clip(np.round(z + 1.5), 0, 4)
    kw = dict(groupCol="query", numIterations=10, numTasks=1, minDataInLeaf=5, evalAt=[1, 3])
    md = LightGBMRanker(**kw).fit(_frame(X, {"label": rel, "query": q}))
    ms = LightGBMRanker(**kw).fit(_frame(sp.csr_matrix(X), {"label": rel, "query": q}))
    assert _model_string(ms) == _model_string(md)
    assert _model_string(LightGBMRanker(matrixType="sparse", **kw).fit(_frame(X, {"label": rel, "query": q}))) == _model_string(md)
    _check_transform(ms, X, ["prediction"], {"prediction": ms.predict})


def test_bundled_one_hot_sparse_fit(built):
    """one-hot blocks fitted from CSR are bundled into shared storage columns, and the model is the dense column's"""
    from mmlspark_b200.lightgbm import LightGBMRegressor
    rng = np.random.default_rng(5)
    n = 5000
    blocks = []
    for levels in (40, 25):
        k = rng.integers(0, levels, n)
        b = np.zeros((n, levels)); b[np.arange(n), k] = 1.0
        blocks.append(b)
    X = np.hstack(blocks + [rng.standard_normal((n, 2))])
    z = X[:, 3] * 2 - X[:, 41] + X[:, 65] + 0.3 * rng.standard_normal(n)
    seen = []

    class Spy(LightGBMRegressor):
        def _make_dataset(self, part, params_str, reference=None):
            ds = super()._make_dataset(part, params_str, reference=reference)
            seen.append(ds.bundles()[0])
            return ds

    ms = Spy(numIterations=8, numTasks=1, minDataInLeaf=5).fit(_frame(sp.csr_matrix(X), {"label": z}))
    assert seen and seen[0] < X.shape[1]
    md = LightGBMRegressor(numIterations=8, numTasks=1, minDataInLeaf=5).fit(_frame(X, {"label": z}))
    assert _model_string(ms) == _model_string(md)
    _check_transform(ms, X, ["prediction"], {"prediction": ms.predict})


def test_validation_early_stopping_and_batches_sparse(built):
    from mmlspark_b200.lightgbm import LightGBMClassifier
    rng, X, z = _data(6, n=6000)
    y = (z + rng.standard_normal(len(z)) > np.median(z)).astype(np.float64)
    valid = rng.random(len(y)) < 0.25
    kw = dict(numIterations=200, numTasks=1, minDataInLeaf=5, earlyStoppingRound=5, validationIndicatorCol="valid", learningRate=0.3)
    md = LightGBMClassifier(**kw).fit(_frame(X, {"label": y, "valid": valid}))
    ms = LightGBMClassifier(**kw).fit(_frame(sp.csr_matrix(X), {"label": y, "valid": valid}))
    assert ms.getBoosterBestIteration() == md.getBoosterBestIteration() and 0 < md.getBoosterBestIteration() < 200
    assert _model_string(ms) == _model_string(md)
    kb = dict(numIterations=6, numTasks=1, minDataInLeaf=5, numBatches=2)
    bd = LightGBMClassifier(**kb).fit(_frame(X, {"label": y}))
    bs = LightGBMClassifier(**kb).fit(_frame(sp.csr_matrix(X), {"label": y}))
    assert bs.getBoosterNumTotalIterations() == 12 and _model_string(bs) == _model_string(bd)


def test_two_tasks_sparse(built):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200.lightgbm import LightGBMClassifier
    _, X, z = _data(7, n=4000)
    y = (z > np.median(z)).astype(np.float64)
    # the two tasks get the same 4000 rows: the driver numbers ranks in the order the tasks reach it, and each rank finds the bins of
    # a slice of the features on its own shard, so with different shards the two fits would agree only when their tasks arrive in
    # the same order
    X, y = np.vstack([X, X]), np.concatenate([y, y])
    md = LightGBMClassifier(numIterations=10, numTasks=2, defaultListenPort=25400).fit(_frame(X, {"label": y}))
    ms = LightGBMClassifier(numIterations=10, numTasks=2, defaultListenPort=25500).fit(_frame(sp.csr_matrix(X), {"label": y}))
    assert _model_string(ms) == _model_string(md)
    np.testing.assert_array_equal(ms.transform(_frame(sp.csr_matrix(X), {}))["probability"], md.transform(_frame(X, {}))["probability"])


def test_wide_hashed_fit_and_transform_never_densify(built, monkeypatch):
    """2^18 hashed columns x 50K rows would be 105 GB dense: the fit and transform must stay on CSR"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import LightGBMClassifier

    def refuse(*a, **k):
        raise AssertionError("densified")
    monkeypatch.setattr(sp.csr_matrix, "toarray", refuse)
    monkeypatch.setattr(sp.csr_matrix, "todense", refuse)
    monkeypatch.setattr(capi.Dataset, "from_mat", refuse)
    monkeypatch.setattr(capi.Booster, "predict_device", refuse)
    rng = np.random.default_rng(29)
    n, F, per_row = 50_000, 1 << 18, 12
    cols = np.sort(rng.integers(0, 4000, (n, per_row)), axis=1) + np.arange(per_row)[None, :] * 4000
    data = rng.standard_normal(n * per_row)
    X = sp.csr_matrix((data, cols.reshape(-1), np.arange(n + 1) * per_row), shape=(n, F))
    y = (data.reshape(n, per_row)[:, :3].sum(axis=1) > 0).astype(np.float64)
    m = LightGBMClassifier(numIterations=10, numTasks=1, minDataInLeaf=5, leafPredictionCol="leaf").fit(_frame(X, {"label": y}))
    out = m.transform(_frame(X, {}))
    assert out["probability"].shape == (n, 2) and out["leaf"].shape == (n, 10)
    assert out["probability"][y == 1, 1].mean() > out["probability"][y == 0, 1].mean()
    for r in rng.choice(n, 20, replace=False):
        np.testing.assert_array_equal(m.booster.score(X[r], False, True), out["probability"][r])
