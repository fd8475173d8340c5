"""Single-dataset mode: one dataset from several row parts (LGBM_DatasetCreateFromMats, B200GBM_DatasetCreateFromCSRs) and the estimators'
useSingleDatasetMode, where the tasks that share a GPU train as one rank over their partitions.

A multi-part dataset must be the dataset of the concatenated rows, bit for bit: bins, bundles and mappers, and so the model trained on it.
In single-dataset mode a fit with numTasks = 4 on one device must give the native model of numTasks = 1 on the same frame."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import test_gpu_bundling as B
import test_gpu_multi as M
import test_gpu_wide as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DS_PARAMS = M.DS_PARAMS
gpu = pytest.mark.gpu


def _splits(n, sizes):
    """row slices of the given sizes, the last one taking the rest"""
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    assert offs[-1] < n
    offs = np.append(offs, n)
    return [slice(int(offs[i]), int(offs[i + 1])) for i in range(len(offs) - 1)]


def _from_mats_raw(capi, ptrs, nrows, ncol, dtype_code, params, reference=None):
    """LGBM_DatasetCreateFromMats on raw pointers (host or device)"""
    h = C.c_void_p()
    nrow = np.asarray(nrows, dtype=np.int32)
    arr = (C.c_void_p * max(len(ptrs), 1))(*[p if isinstance(p, int) else None for p in ptrs])
    capi.check(capi.load().LGBM_DatasetCreateFromMats(C.c_int32(len(ptrs)), arr, C.c_int(dtype_code), capi._ptr(nrow), C.c_int32(ncol), C.c_int(1),
                                                      params.encode(), reference.handle if reference is not None else None, C.byref(h)))
    return capi.Dataset(h)


def _train(capi, ds, y, params, iters=6):
    ds.set_field("label", y)
    b = capi.Booster(ds, params)
    try:
        for _ in range(iters):
            if b.update_one_iter():
                break
        return b.save_model_to_string()
    finally:
        b.free()


def _assert_same_dataset(a, b, wide=False, mappers=True):
    assert a.num_data() == b.num_data() and a.num_feature() == b.num_feature()
    if wide:
        assert np.array_equal(a.get_bins16(), b.get_bins16())
    else:
        assert np.array_equal(a.get_bins(), b.get_bins())
    ka, ca = a.bundles()
    kb, cb = b.bundles()
    assert ka == kb and np.array_equal(ca, cb)
    if mappers:
        for f in range(a.num_feature()):
            assert a.feature_info(f) == b.feature_info(f)
            assert a.upper_bounds(f).tobytes() == b.upper_bounds(f).tobytes()


# ------------------------------------------------------------------------------------------------ C ABI, dense
def _dense_case(case):
    """(X, y, dataset params, training params, part sizes)"""
    rng = np.random.default_rng({"f32": 1, "f64": 2, "device": 3, "bundle": 4, "wide": 5, "chunks": 6}[case])
    if case == "bundle":
        X, z = B._one_hot_data(41, 20_000)
        return X, z.astype(np.float32), B.DS, M._params("regression", 1), [7000, 1, 6000]
    if case == "wide":
        X, s = W._data(42, 30_000)
        return X, (s > 0).astype(np.float32), W.DS, W._params("binary", "is_unbalance=false"), [9000, 1, 11000]
    if case == "chunks":      # 4096 f64 columns: a 256 MB staging chunk holds 8192 rows, so every part spans several chunks
        n, F = 39_001, 4096
        X = rng.integers(0, 40, (n, F)).astype(np.float64)
        X[rng.random((n, F)) < 0.01] = np.nan
        y = (X[:, 0] + np.nan_to_num(X[:, 1]) * 0.5 - X[:, 2] + rng.standard_normal(n)).astype(np.float32)
        return X, y, DS_PARAMS, M._params("regression", 1, "num_leaves=15"), [12_000, 17_000]
    n, F = 24_000, 25
    X = rng.standard_normal((n, F))
    X[:, 4] = np.where(rng.random(n) < 0.2, np.nan, X[:, 4])
    X[:, 6] = np.where(rng.random(n) < 0.8, 0.0, X[:, 6])
    y = (1.5 * X[:, 0] + np.sin(2 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.3 * rng.standard_normal(n)).astype(np.float32)
    if case == "f32":
        X = X.astype(np.float32)
    return X, y, DS_PARAMS, M._params("regression", 1), [5000, 1, 9000]


@gpu
@pytest.mark.parametrize("case", ["f32", "f64", "device", "bundle", "wide", "chunks"])
def test_from_mats_equals_from_mat_of_the_concatenation(built, case):
    from mmlspark_b200 import capi
    X, y, ds_params, params, sizes = _dense_case(case)
    parts = [np.ascontiguousarray(X[sl]) for sl in _splits(len(X), sizes)]
    assert any(len(p) == 1 for p in parts) or case == "chunks"
    whole = capi.Dataset.from_mat(X, ds_params)
    bufs = []
    try:
        if case == "device":      # part 2 lives in device memory, the others on the host
            buf = capi.DeviceBuffer(parts[2].nbytes)
            bufs.append(buf)
            capi.memcpy(buf.ptr, parts[2].ctypes.data, parts[2].nbytes)
            ptrs = [p.ctypes.data for p in parts]
            ptrs[2] = buf.ptr.value
            multi = _from_mats_raw(capi, ptrs, [len(p) for p in parts], X.shape[1], capi.DTYPE_FLOAT64, ds_params)
        else:
            multi = capi.Dataset.from_mats(parts, ds_params)
        if case == "bundle":
            assert multi.bundles()[0] < X.shape[1], "no bundle formed"
        if case == "chunks":
            assert multi.ingest_ms() > 0
        _assert_same_dataset(multi, whole, wide=case == "wide", mappers=case != "chunks")
        assert _train(capi, multi, y, params) == _train(capi, whole, y, params)
        multi.free()
    finally:
        for buf in bufs:
            buf.free()
        whole.free()


@gpu
def test_from_mats_validation_data_uses_the_reference_bins(built):
    from mmlspark_b200 import capi
    X, y, ds_params, _, sizes = _dense_case("f64")
    train = capi.Dataset.from_mats([X[sl] for sl in _splits(len(X), sizes)], ds_params)
    Xv = np.random.default_rng(9).standard_normal((3001, X.shape[1])) * 1.3
    a = capi.Dataset.from_mats([Xv[:1000], Xv[1000:1001], Xv[1001:]], ds_params, reference=train)
    b = capi.Dataset.from_mat(Xv, ds_params, reference=train)
    _assert_same_dataset(a, b)
    for ds in (a, b, train):
        ds.free()


# ------------------------------------------------------------------------------------------------ C ABI, CSR
def _csr_parts(indptr, indices, data, splits, rebase):
    """CSR row parts of one CSR: with rebase=False each part keeps the whole indices / data and its slice of indptr, which then does not
    start at 0; with rebase=True a part holds its own elements and an indptr from 0"""
    out = []
    for i, sl in enumerate(splits):
        ip = indptr[sl.start:sl.stop + 1].astype(np.int64)
        if rebase and i % 2 == 0:
            a, b = int(ip[0]), int(ip[-1])
            out.append((ip - a, indices[a:b], data[a:b]))
        else:
            out.append((ip, indices, data))
    return out


@gpu
@pytest.mark.parametrize("case", ["random", "bundle"])
def test_from_csrs_equals_from_csr_of_the_concatenation(built, case):
    from mmlspark_b200 import capi
    import test_gpu_ingest_scale as I
    rng = np.random.default_rng(11)
    if case == "bundle":
        X, z = B._one_hot_data(43, 20_000)
        indptr, indices, data = B._csr(X)
        y, ds_params, params = z.astype(np.float32), B.DS, M._params("regression", 1)
    else:
        X, indptr, indices, data = I._random_csr(rng, 30_000, 40, 0.15)
        y = (np.nan_to_num(X[:, 0]) * 2 - np.nan_to_num(X[:, 1]) + 0.1 * rng.standard_normal(len(X)) > 0).astype(np.float32)
        ds_params, params = DS_PARAMS, M._params("binary", 1, "is_unbalance=false")
    F = X.shape[1]
    whole = capi.Dataset.from_csr(indptr, indices, data, F, ds_params)
    splits = _splits(len(X), [6000, 1, 8000])
    for rebase in (False, True):
        multi = capi.Dataset.from_csrs(_csr_parts(indptr, indices, data, splits, rebase), F, ds_params)
        if case == "bundle":
            assert multi.bundles()[0] < F, "no bundle formed"
        _assert_same_dataset(multi, whole)
        assert _train(capi, multi, y, params) == _train(capi, whole, y, params)
        multi.free()
    # scipy matrices as parts, and validation data with reference=
    import scipy.sparse as sp
    m = sp.csr_matrix((data, indices, indptr), shape=X.shape)
    multi = capi.Dataset.from_csrs([m[sl] for sl in splits], F, ds_params)
    _assert_same_dataset(multi, whole, mappers=False)
    va = capi.Dataset.from_csrs([m[:500], m[500:2000]], F, ds_params, reference=multi)
    vb = capi.Dataset.from_csr(m[:2000].indptr, m[:2000].indices, m[:2000].data, F, ds_params, reference=whole)
    _assert_same_dataset(va, vb, mappers=False)
    for ds in (va, vb, multi, whole):
        ds.free()


@gpu
def test_from_csrs_wide_sparse_does_not_densify(built):
    """2^18 hashed columns in three parts: bins of sampled rows, the storage layout and the trained model equal the one-part CSR's"""
    from mmlspark_b200 import capi
    rng = np.random.default_rng(29)
    n, F, per_row = 30_000, 1 << 18, 8
    cols = np.sort(rng.integers(0, 150, (n, per_row)), axis=1) + np.arange(per_row)[None, :] * 30_000
    indices = cols.reshape(-1).astype(np.int32)
    indptr = (np.arange(n + 1) * per_row).astype(np.int64)
    data = rng.standard_normal(n * per_row)
    y = (data.reshape(n, per_row)[:, 0] + 0.3 * rng.standard_normal(n) > 0).astype(np.float32)
    params_ds = DS_PARAMS + " min_data_in_leaf=5"
    whole = capi.Dataset.from_csr(indptr.astype(np.int32), indices, data, F, params_ds)
    multi = capi.Dataset.from_csrs(_csr_parts(indptr, indices, data, _splits(n, [10_000, 9_999]), True), F, params_ds)
    rows = np.sort(rng.choice(n, 2000, replace=False)).astype(np.int32)
    assert np.array_equal(multi.get_bins_rows(rows), whole.get_bins_rows(rows))
    ka, ca = multi.bundles()
    kb, cb = whole.bundles()
    assert ka == kb and np.array_equal(ca, cb)
    params = M._params("binary", 1, "is_unbalance=false min_data_in_leaf=5")
    assert _train(capi, multi, y, params, 4) == _train(capi, whole, y, params, 4)
    multi.free(); whole.free()


# ------------------------------------------------------------------------------------------------ errors
@gpu
def test_rejected_inputs_fail_with_a_message_and_leave_the_library_usable(built):
    from mmlspark_b200 import capi
    X = np.random.default_rng(3).standard_normal((300, 5))
    err = lambda: capi.load().LGBM_GetLastError().decode()      # noqa: E731
    with pytest.raises(capi.LightGBMError, match="nmat"):
        _from_mats_raw(capi, [], [], 5, capi.DTYPE_FLOAT64, DS_PARAMS)
    with pytest.raises(capi.LightGBMError, match=r"at least one row.*part 1"):
        _from_mats_raw(capi, [X.ctypes.data, X.ctypes.data], [300, 0], 5, capi.DTYPE_FLOAT64, DS_PARAMS)
    with pytest.raises(capi.LightGBMError, match=r"null.*part 1"):
        _from_mats_raw(capi, [X.ctypes.data, None], [300, 10], 5, capi.DTYPE_FLOAT64, DS_PARAMS)
    h = C.c_void_p()
    assert capi.load().LGBM_DatasetCreateFromMats(C.c_int32(2), None, C.c_int(1), None, C.c_int32(5), C.c_int(1), b"", None, C.byref(h)) == -1
    assert "null" in err()
    ip = np.array([0, 2, 4, 6], dtype=np.int64)
    ix = np.array([0, 1, 2, 3, 4, 0], dtype=np.int32)
    v = np.ones(6)
    good = (ip, ix, v)
    with pytest.raises(capi.LightGBMError, match=r"non-decreasing.*part 1"):
        capi.Dataset.from_csrs([good, (np.array([0, 4, 2, 6]), ix, v)], 5, DS_PARAMS)
    with pytest.raises(capi.LightGBMError, match=r"number of elements.*part 2"):
        capi.Dataset.from_csrs([good, good, (np.array([0, 2, 7]), ix, v)], 5, DS_PARAMS)
    with pytest.raises(capi.LightGBMError, match=r"number of elements.*part 0"):
        capi.Dataset.from_csrs([(np.array([-1, 2]), ix, v), good], 5, DS_PARAMS)
    with pytest.raises(capi.LightGBMError, match=r"column index.*part 1"):
        capi.Dataset.from_csrs([good, (ip, np.array([0, 1, 2, 3, 9, 0], dtype=np.int32), v)], 5, DS_PARAMS)
    with pytest.raises(capi.LightGBMError, match=r"at least one row.*part 1"):
        capi.Dataset.from_csrs([good, (np.array([3]), ix, v)], 5, DS_PARAMS)
    assert capi.load().B200GBM_DatasetCreateFromCSRs(C.c_int32(0), None, C.c_int(3), None, None, C.c_int(1), None, None, C.c_int64(5), b"",
                                                     None, C.byref(h)) == -1
    assert "nparts" in err()
    # still usable
    ds = capi.Dataset.from_mats([X[:100], X[100:]], DS_PARAMS)
    ref = capi.Dataset.from_mat(X, DS_PARAMS)
    assert np.array_equal(ds.get_bins(), ref.get_bins())
    ds.free(); ref.free()


def test_new_entries_are_declared_and_exported(built):
    from mmlspark_b200 import capi
    txt = open(os.path.join(ROOT, "include", "b200gbm_c_api.h")).read()
    for name in ("LGBM_DatasetCreateFromMats", "B200GBM_DatasetCreateFromCSRs"):
        assert re.search(r"\bint %s\(" % name, txt), name
        assert hasattr(capi.load(), name), name
    assert "[UPSTREAM] LightGBM's LGBM_DatasetCreateFromMats" in txt


# ------------------------------------------------------------------------------------------------ estimators, task groups (no GPU)
def test_device_groups_and_main_tasks(monkeypatch):
    from mmlspark_b200.lightgbm import LightGBMRegressor
    from mmlspark_b200.lightgbm.estimators import LightGBMBase
    est = LightGBMRegressor(useSingleDatasetMode=True)
    parts = [slice(0, 10), slice(10, 20), slice(20, 30), slice(30, 40), slice(40, 50)]
    monkeypatch.setattr(LightGBMBase, "_num_devices", lambda self: 2)
    assert [est._device_group(p, parts, 5) for p in range(5)] == [[0, 2, 4], [1, 3], [], [], []]
    parts[0] = slice(0, 0)      # an empty partition hands the group to the next pid
    assert [est._device_group(p, parts, 5) for p in range(5)] == [[], [1, 3], [2, 4], [], []]
    monkeypatch.setattr(LightGBMBase, "_num_devices", lambda self: 1)
    assert [est._device_group(p, parts, 5) for p in range(5)] == [[], [1, 2, 3, 4], [], [], []]


# ------------------------------------------------------------------------------------------------ estimators, one device
def _fit_counting(monkeypatch, est, df):
    """fit, and return (model, network_init calls, boosters the tasks returned)"""
    from mmlspark_b200.lightgbm import estimators as ES
    from mmlspark_b200.lightgbm import train_utils as tu
    calls, returned = [], []
    real_init, real_train = tu.network_init, ES.LightGBMBase._train_lightgbm

    def counting_init(*a, **k):
        calls.append(a)
        return real_init(*a, **k)

    def recording_train(self, *a, **k):
        r = real_train(self, *a, **k)
        returned.append(r)
        return r
    monkeypatch.setattr(tu, "network_init", counting_init)
    monkeypatch.setattr(ES.LightGBMBase, "_train_lightgbm", recording_train)
    try:
        return est.fit(df), len(calls), [r for r in returned if r is not None]
    finally:
        monkeypatch.setattr(tu, "network_init", real_init)
        monkeypatch.setattr(ES.LightGBMBase, "_train_lightgbm", real_train)


def _estimator_case(case):
    from mmlspark_b200.lightgbm import Frame, LightGBMClassifier, LightGBMRanker, LightGBMRegressor
    rng = np.random.default_rng(["binary", "multiclass", "regressor", "ranker", "sparse", "valid", "batches"].index(case))
    n, F = 12_000, 10
    X = rng.standard_normal((n, F))
    X[:, 5] = np.where(rng.random(n) < 0.7, 0.0, X[:, 5])
    s = X[:, 0] + 0.8 * X[:, 1] * X[:, 2] + 0.5 * np.sin(3 * X[:, 3]) + 0.5 * rng.standard_normal(n)
    if case == "multiclass":
        K = 3
        y = np.digitize(s, np.quantile(s, [1 / 3, 2 / 3])).astype(np.float64)
        init = 0.1 * rng.standard_normal((n, K))
        return LightGBMClassifier, dict(objective="multiclass", initScoreCol="init"), Frame({"features": X, "label": y, "init": init})
    if case == "regressor":
        return LightGBMRegressor, dict(weightCol="w"), Frame({"features": X, "label": s, "w": rng.random(n) + 0.5})
    if case == "ranker":
        q = np.repeat(np.arange(600), 20)[:n]
        rel = np.clip(np.round(s + 1.5), 0, 4)
        perm = rng.permutation(n)
        return LightGBMRanker, dict(groupCol="query", minDataInLeaf=5), Frame({"features": X[perm], "label": rel[perm], "query": q[perm]})
    y = (s > 0).astype(np.float64)
    df = Frame({"features": X, "label": y})
    if case == "sparse":
        return LightGBMClassifier, dict(matrixType="sparse"), df
    if case == "valid":
        df = df.with_column("valid", rng.random(n) < 0.3)
        return LightGBMClassifier, dict(validationIndicatorCol="valid", earlyStoppingRound=3, learningRate=0.3, numLeaves=63, metric="auc"), df
    if case == "batches":
        return LightGBMClassifier, dict(numBatches=2), df
    return LightGBMClassifier, {}, df


@gpu
@pytest.mark.parametrize("case", ["binary", "multiclass", "regressor", "ranker", "sparse", "valid", "batches"])
def test_four_tasks_on_one_device_train_the_one_task_model(built, monkeypatch, case):
    from mmlspark_b200.lightgbm.estimators import LightGBMBase
    monkeypatch.setattr(LightGBMBase, "_num_devices", lambda self: 1)
    cls, kw, df = _estimator_case(case)
    iters = 200 if case == "valid" else 8
    one, _, _ = _fit_counting(monkeypatch, cls(numIterations=iters, numTasks=1, **kw), df)
    four, inits, boosters = _fit_counting(monkeypatch, cls(numIterations=iters, numTasks=4, useSingleDatasetMode=True, defaultListenPort=27100, **kw), df)
    assert inits == 0 and len(boosters) == max(kw.get("numBatches", 0), 1)      # one booster per batch
    assert four.getNativeModel() == one.getNativeModel()
    assert four.getBoosterBestIteration() == one.getBoosterBestIteration()
    if case == "valid":
        assert 0 < one.getBoosterNumTotalIterations() < iters
    if case == "batches":
        assert one.getBoosterNumTotalIterations() == 2 * iters


# ------------------------------------------------------------------------------------------------ estimators, two devices emulated on one
@gpu
def test_two_device_groups_train_through_the_same_device_collective(built, monkeypatch):
    """numTasks = 4 over 2 (emulated) devices: the main tasks 0 and 1 train as two ranks on p0+p2 and p1+p3"""
    from mmlspark_b200 import capi
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    from mmlspark_b200.lightgbm.estimators import LightGBMBase
    from mmlspark_b200.lightgbm.params import dataset_params
    from mmlspark_b200.modeltext import parse_model, compare_models
    from oracle import oracle as O
    real = capi.set_device
    monkeypatch.setattr(capi, "set_device", lambda ordinal: real(0))
    monkeypatch.setattr(LightGBMBase, "_num_devices", lambda self: 2)
    rng = np.random.default_rng(77)
    n, F = 40_003, 16
    X = rng.standard_normal((n, F))
    y = 1.5 * X[:, 0] + np.sin(2 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.3 * rng.standard_normal(n)
    df = Frame({"features": X, "label": y})
    est = LightGBMRegressor(numIterations=8, numTasks=4, useSingleDatasetMode=True, defaultListenPort=27200)
    model, inits, boosters = _fit_counting(monkeypatch, est, df)
    assert inits == 2 and len(boosters) == 1
    p = est._partitions(df, 4)
    groups = [[p[0], p[2]], [p[1], p[3]]]
    params = est.getTrainParams(4, df).to_string().replace("num_machines=4", "num_machines=2")
    ds_params = dataset_params(255, 200000, 0)
    last = None
    for order in (groups, groups[::-1]):      # the driver numbers ranks in arrival order
        rows = np.concatenate([np.arange(sl.start, sl.stop) for g in order for sl in g])
        ods = O.OracleDataset(X[rows], ds_params, rank_rows=[sum(sl.stop - sl.start for sl in g) for g in order])
        ods.set_field("label", y[rows].astype(np.float32))
        ob = O.OracleBooster(ods, params)
        ob.train(8)
        try:
            compare_models(parse_model(model.getNativeModel()), parse_model(ob.model_string()))
            return
        except AssertionError as e:
            last = e
    raise last


# ------------------------------------------------------------------------------------------------ two real GPUs
@gpu
def test_three_tasks_on_two_gpus_train_in_single_dataset_mode(built):
    if M._ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from mmlspark_b200.lightgbm import LightGBMClassifier
    from mmlspark_b200.lightgbm.estimators import LightGBMBase
    if LightGBMBase._num_devices(None) != 2:
        pytest.skip("needs exactly 2 GPUs for the mixed layout")
    _, _, df = _estimator_case("binary")
    m = LightGBMClassifier(numIterations=10, numTasks=3, useSingleDatasetMode=True, defaultListenPort=27300).fit(df)
    assert m.getBoosterNumTotalIterations() == 10
