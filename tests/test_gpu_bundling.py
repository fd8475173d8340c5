"""Exclusive feature bundling: mutually exclusive sparse features share one uint8 storage column, and training on the bundled dataset
is identical to training with enable_bundle=false — the same trees byte for byte, the same training and validation scores and metrics
bit for bit.  Also: a conflict outside the bin-construction sample dissolves its bundle, the bins and the histogram entry read back per
feature exactly as without bundles, and dense data forms no bundle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS = "max_bin=255 min_data_in_leaf=5 is_pre_partition=True num_threads=0"


def _one_hot_data(seed, n):
    """one-hot blocks, dense columns, sparse features with NaN, with negatives (most frequent bin in the middle) and non-negative ones"""
    rng = np.random.default_rng(seed)
    cols = []
    for levels in (40, 25, 12):
        k = rng.integers(0, levels, n)
        block = np.zeros((n, levels)); block[np.arange(n), k] = 1.0
        cols.append(block)
    cols.append(rng.standard_normal((n, 3)))
    owner = rng.integers(0, 30, n)          # the 12 sparse features are mutually exclusive: at most one is non-zero in a row
    for i, kind in enumerate(k for k in ("nan", "neg", "pos") for _ in range(4)):
        v = np.zeros(n)
        on = owner == i
        if kind == "nan":
            v[on] = np.where(rng.random(on.sum()) < 0.5, np.nan, rng.standard_normal(on.sum()))
        elif kind == "neg":
            v[on] = rng.standard_normal(on.sum()) * 3
        else:
            v[on] = rng.random(on.sum()) * 5 + 0.1
        cols.append(v[:, None])
    X = np.hstack(cols)
    z = X[:, 3] * 2 - X[:, 40] + X[:, 66] * 1.5 + np.nan_to_num(X[:, 80]) + np.nan_to_num(X[:, 85]) * 0.7 + 0.3 * rng.standard_normal(n)
    return X, z


NAN_FEATURES, NEG_FEATURES = range(80, 84), range(84, 88)     # sparse members with a NaN bin / with the most frequent bin in the middle


def _shares_column(column_of, features):
    """some feature of `features` shares its storage column with another feature"""
    return any((column_of == column_of[f]).sum() > 1 for f in features)


def _csr(X):
    stored = (X != 0) | np.isnan(X)
    indptr = np.concatenate([[0], np.cumsum(stored.sum(axis=1))]).astype(np.int32)
    return indptr, np.nonzero(stored)[1].astype(np.int32), X[stored]


def _labels(z, objective):
    if objective == "binary":
        return (z > np.median(z)).astype(np.float64)
    if objective == "multiclass":
        return np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])).astype(np.float64)
    return z


def _datasets(capi, X, Xv, y, yv, params, fmt):
    if fmt == "csr":
        tr = capi.Dataset.from_csr(*_csr(X), X.shape[1], params)
        va = capi.Dataset.from_csr(*_csr(Xv), Xv.shape[1], params, reference=tr)
    else:
        tr = capi.Dataset.from_mat(X, params, row_major=(fmt != "mat_col"))
        va = capi.Dataset.from_mat(Xv, params, reference=tr, row_major=(fmt != "mat_col"))
    tr.set_field("label", y); va.set_field("label", yv)
    return tr, va


def _train(capi, X, Xv, y, yv, ds_params, params, fmt, iters=8):
    tr, va = _datasets(capi, X, Xv, y, yv, ds_params, fmt)
    b = capi.Booster(tr, params)
    b.add_valid(va)
    evals = []
    for _ in range(iters):
        b.update_one_iter()
        evals.append((b.get_eval(0).copy(), b.get_eval(1).copy()))
    model = b.save_model_to_string()
    out = dict(trees=model.split("\nparameters:")[0], scores=b.get_scores(0), vscores=b.get_scores(1), evals=evals, bundles=tr.bundles())
    b.free(); tr.free(); va.free()
    return out


CONFIGS = {
    "binary": "objective=binary metric=binary_logloss,auc num_leaves=15",
    "multiclass": "objective=multiclass num_class=3 metric=multi_logloss num_leaves=7",
    "l1": "objective=regression_l1 metric=l1 num_leaves=15",
    "feature_fraction": "objective=regression metric=l2 num_leaves=15 feature_fraction=0.5",
    "bagging": "objective=binary metric=binary_logloss num_leaves=15 bagging_fraction=0.7 bagging_freq=1",
    "goss": "objective=binary metric=binary_logloss num_leaves=15 boosting=goss learning_rate=0.3",
    "dart": "objective=regression metric=l2 num_leaves=15 boosting=dart drop_rate=0.5 skip_drop=0",
    "max_depth": "objective=regression metric=l2 num_leaves=31 max_depth=3",
}


@pytest.mark.parametrize("fmt", ["mat", "mat_col", "csr"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_bundled_training_equals_unbundled(built, config, fmt):
    from mmlspark_b200 import capi
    X, z = _one_hot_data(1, 6000)
    Xv, zv = _one_hot_data(2, 2000)
    obj = "binary" if "binary" in CONFIGS[config] else ("multiclass" if "multiclass" in CONFIGS[config] else "regression")
    y, yv = _labels(z, obj), _labels(zv, obj)
    params = DS + " " + CONFIGS[config]
    a = _train(capi, X, Xv, y, yv, DS, params, fmt)
    b = _train(capi, X, Xv, y, yv, DS + " enable_bundle=false", params + " enable_bundle=false", fmt)
    ncols, column_of = a["bundles"]
    assert ncols < 0.3 * X.shape[1], ncols
    assert _shares_column(column_of, NAN_FEATURES) and _shares_column(column_of, NEG_FEATURES), column_of
    assert b["bundles"][0] == int((b["bundles"][1] >= 0).sum())
    assert a["trees"] == b["trees"]
    assert np.array_equal(a["scores"], b["scores"]) and np.array_equal(a["vscores"], b["vscores"])
    for (ta, va), (tb, vb) in zip(a["evals"], b["evals"]):
        assert np.array_equal(ta, tb) and np.array_equal(va, vb)


def test_bundled_training_without_column_copy(built, monkeypatch):
    from mmlspark_b200 import capi
    monkeypatch.setenv("B200GBM_COLUMN_COPY", "0")
    X, z = _one_hot_data(3, 5000)
    Xv, zv = _one_hot_data(4, 1000)
    params = DS + " objective=regression metric=l2 num_leaves=15"
    a = _train(capi, X, Xv, z, zv, DS, params, "mat")
    b = _train(capi, X, Xv, z, zv, DS + " enable_bundle=false", params + " enable_bundle=false", "mat")
    assert a["bundles"][0] < b["bundles"][0]
    assert a["trees"] == b["trees"] and np.array_equal(a["vscores"], b["vscores"])


@pytest.mark.parametrize("fmt", ["mat", "csr"])
def test_conflict_outside_the_sample_dissolves_the_bundle(built, fmt):
    """features 0/1 are exclusive on the sampled rows but both non-zero on an unsampled row; 2/3 are exclusive on every row"""
    from mmlspark_b200 import capi
    n, k = 4000, 800
    rng = np.random.default_rng(7)
    sampled = capi.sample_indices(n, k, 1)
    unsampled = np.setdiff1d(np.arange(n), sampled)
    X = np.zeros((n, 5))
    X[:, 4] = rng.standard_normal(n)
    half = len(sampled) // 2
    for f, rows in ((0, sampled[:half]), (1, sampled[half:]), (2, sampled[:half]), (3, sampled[half:])):
        X[rows[::3], f] = rng.random(len(rows[::3])) + 0.5
    for f, rows in ((0, unsampled[:1000]), (1, unsampled[999:2000]), (2, unsampled[:1000]), (3, unsampled[1000:2000])):
        X[rows[::2], f] = rng.random(len(rows[::2])) + 0.5
    X[unsampled[1000], 0] = X[unsampled[1000], 1] = 2.0          # the one conflicting row: not in the sample
    assert X[unsampled[1000], 0] != 0 and X[unsampled[1000], 1] != 0
    assert not ((X[:, 2] != 0) & (X[:, 3] != 0)).any()
    y = X[:, 0] - X[:, 1] + 0.5 * X[:, 2] + X[:, 3] + X[:, 4] + 0.1 * rng.standard_normal(n)
    ds_params = DS + f" bin_construct_sample_cnt={k}"
    Xv = X[:500]
    params = ds_params + " objective=regression metric=l2 num_leaves=7"
    a = _train(capi, X, Xv, y, y[:500], ds_params, params, fmt)
    b = _train(capi, X, Xv, y, y[:500], ds_params + " enable_bundle=false", params + " enable_bundle=false", fmt)
    ncols, col = a["bundles"]
    assert col[2] == col[3], col
    assert col[0] != col[1], col
    assert ncols == 4
    assert a["trees"] == b["trees"] and np.array_equal(a["scores"], b["scores"]) and np.array_equal(a["vscores"], b["vscores"])


@pytest.mark.parametrize("fmt", ["mat", "csr"])
def test_bins_and_histogram_read_back_per_feature(built, fmt):
    from mmlspark_b200 import capi
    X, z = _one_hot_data(5, 3000)
    zero = np.nonzero(X[:, 88] == 0)[0][:5]
    X[zero, 88] = -np.inf          # most frequent bin 0 of a positive-only member: -inf lands there, and stays at slot 0
    if fmt == "csr":
        a = capi.Dataset.from_csr(*_csr(X), X.shape[1], DS)
        b = capi.Dataset.from_csr(*_csr(X), X.shape[1], DS + " enable_bundle=false")
    else:
        a = capi.Dataset.from_mat(X, DS)
        b = capi.Dataset.from_mat(X, DS + " enable_bundle=false")
    assert a.bundles()[0] < b.bundles()[0]
    assert np.array_equal(a.get_bins(), b.get_bins())
    rows = np.array([0, 5, 17, 1000, 2999], dtype=np.int32)
    assert np.array_equal(a.get_bins_rows(rows), b.get_bins_rows(rows))
    rng = np.random.default_rng(6)
    g = rng.standard_normal(3000).astype(np.float32); h = (rng.random(3000) + 0.1).astype(np.float32)
    idx = np.sort(rng.choice(3000, 1200, replace=False)).astype(np.int32)
    assert np.array_equal(a.histogram(g, h), b.histogram(g, h))
    assert np.array_equal(a.histogram(g, h, idx), b.histogram(g, h, idx))
    a.free(); b.free()


def test_dense_data_forms_no_bundle(built):
    """dense columns and a 30 %-dense quarter (as in the benchmark's sparse configuration) conflict on most rows: every column stays plain"""
    from mmlspark_b200 import capi
    rng = np.random.default_rng(8)
    n, F = 20000, 64
    X = rng.standard_normal((n, F)).astype(np.float32)
    X[:, F // 2:F // 2 + F // 4] *= rng.random((n, F // 4)) < 0.3
    ds = capi.Dataset.from_mat(X, DS)
    ncols, col = ds.bundles()
    assert ncols == F and sorted(col.tolist()) == list(range(F))
    ds.free()


def test_bundled_training_matches_the_oracle(built):
    """the bundled CUDA path against the CPU oracle (which never bundles) at the parity bar: tree structure exact, values within 1e-5"""
    from mmlspark_b200 import capi
    from mmlspark_b200.modeltext import compare_models, parse_model
    from oracle import oracle as O
    X, z = _one_hot_data(9, 8000)
    y = _labels(z, "binary")
    ds_params = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
    params = ds_params + " objective=binary num_leaves=15 min_data_in_leaf=20 learning_rate=0.1 metric="
    ds = capi.Dataset.from_mat(X, ds_params)
    ods = O.OracleDataset(X, ds_params)
    ds.set_field("label", y); ods.set_field("label", y)
    ncols, column_of = ds.bundles()
    assert ncols < 0.3 * X.shape[1] and _shares_column(column_of, NEG_FEATURES), column_of
    b = capi.Booster(ds, params)
    ob = O.OracleBooster(ods, params)
    for _ in range(10):
        assert b.update_one_iter() == ob.update()
    compare_models(parse_model(b.save_model_to_string()), parse_model(ob.model_string()))
    b.free(); ds.free()


def _ngpu():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        return len([l for l in out.splitlines() if l.startswith("GPU ")])
    except Exception:
        return 0


def _two_ranks(X, y, fmt, ds_params, params, iters, base_port):
    """tree_learner=data on 2 rank-threads of one process (thread r <-> GPU r <-> NCCL rank r), each with half of the rows"""
    import threading
    from mmlspark_b200 import capi
    machines = "127.0.0.1:%d,127.0.0.1:%d" % (base_port, base_port + 1)
    half = len(X) // 2
    out, errs = [None, None], []

    def task(r):
        try:
            capi.set_device(r)
            capi.network_init(machines, base_port + r, 120, 2)
            Xr, yr = X[r * half:(r + 1) * half], y[r * half:(r + 1) * half]
            ds = capi.Dataset.from_csr(*_csr(Xr), Xr.shape[1], ds_params) if fmt == "csr" else capi.Dataset.from_mat(Xr, ds_params)
            ds.set_field("label", yr)
            b = capi.Booster(ds, params)
            for _ in range(iters):
                b.update_one_iter()
            out[r] = dict(trees=b.save_model_to_string().split("\nparameters:")[0], scores=b.get_scores(0), bundles=ds.bundles())
            b.free(); ds.free()
            capi.network_free()
        except Exception as e:   # noqa
            errs.append((r, repr(e)))

    ts = [threading.Thread(target=task, args=(r,)) for r in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(180)
    assert not errs, errs
    return out


@pytest.mark.parametrize("fmt", ["mat", "csr"])
def test_two_ranks_bundled_equals_unbundled(built, fmt):
    """Data-parallel: rank 0's grouping reaches rank 1, and features 92/93, exclusive on rank 0's rows but both non-zero on one row of
    rank 1, never share a column; every rank has the same layout, and the model equals the unbundled data-parallel one."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    X, z = _one_hot_data(11, 8000)
    rng = np.random.default_rng(12)
    extra = np.zeros((len(X), 2))
    rows = rng.permutation(len(X))[:800]
    extra[rows[:400], 0] = rng.random(400) + 0.5
    extra[rows[400:], 1] = rng.random(400) + 0.5
    r1 = 4000 + int(np.nonzero(extra[4000:, 0] == 0)[0][0])      # a row of rank 1 where feature 92 is zero: make both non-zero there
    extra[r1] = (2.0, 3.0)
    X = np.hstack([X, extra])
    y = _labels(z + extra[:, 0] - extra[:, 1], "binary")
    params = DS + " objective=binary metric=binary_logloss num_leaves=15 tree_learner=data num_machines=2"
    port = 23500 if fmt == "mat" else 23520
    a = _two_ranks(X, y, fmt, DS, params, 8, port)
    b = _two_ranks(X, y, fmt, DS + " enable_bundle=false", params + " enable_bundle=false", 8, port + 10)
    for r in range(2):
        assert np.array_equal(a[r]["bundles"][1], a[0]["bundles"][1]) and a[r]["bundles"][0] == a[0]["bundles"][0]
        assert a[r]["bundles"][0] < b[r]["bundles"][0]
        assert a[r]["bundles"][1][92] != a[r]["bundles"][1][93]
        assert a[r]["trees"] == b[r]["trees"] and np.array_equal(a[r]["scores"], b[r]["scores"])
    assert _shares_column(a[0]["bundles"][1], NAN_FEATURES)
