"""Batched GPU prediction of CSR rows (B200GBM_BoosterPredictForCSRDevice) against the two predictors it must agree with: the dense
batched predictor on the same rows densified (the last of repeated indices wins, indices outside the model's features are dropped),
bit for bit, and LGBM_BoosterPredictForCSRSingle row by row, bit for bit except contributions (to 1e-12, see _assert_like_single).  Every predict type, the full iteration range and a sub-range, on rows with
empty rows, stored zeros and NaN, unsorted and repeated indices, out-of-range and negative indices, and num_col narrower than the model."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS = "max_bin=255 min_data_in_leaf=5 is_pre_partition=True num_threads=0"
RANGES = [(0, -1), (3, 5)]


def _model_data(rng, n, F):
    X = rng.standard_normal((n, F))
    X[rng.random((n, F)) < 0.3] = 0.0
    X[rng.random((n, F)) < 0.05] = np.nan
    z = np.nan_to_num(X[:, 0]) * 2 - np.nan_to_num(X[:, 1]) + np.nan_to_num(X[:, 2]) ** 2 + 0.3 * rng.standard_normal(n)
    return X, z


def _train(capi, X, y, params, ds_params=DS, iters=10):
    ds = capi.Dataset.from_mat(X, ds_params)
    ds.set_field("label", y.astype(np.float32))
    b = capi.Booster(ds, params + " num_leaves=15 learning_rate=0.2 verbosity=-1 min_data_in_leaf=5")
    for _ in range(iters):
        b.update_one_iter()
    return b, ds


def _zero_missing(model_str):
    """the model with every numerical split on an even feature switched to zero-as-missing (missing type 1, decision_type bits 2-3)"""
    out, split = [], None
    for ln in model_str.split("\n"):
        if ln.startswith("split_feature="):
            split = [int(v) for v in ln.split("=")[1].split()]
        if ln.startswith("decision_type="):
            dts = [int(v) for v in ln.split("=")[1].split()]
            ln = "decision_type=" + " ".join(str((d & ~12) | 4 if not d & 1 and f % 2 == 0 else d) for d, f in zip(dts, split))
        out.append(ln)
    return "\n".join(out)


def _assert_like_single(got, single, pt, msg=""):
    """the single-row predictor runs on the host: TreeSHAP there does not fuse multiply-adds as the device kernel (shared with the dense
    batched predictor) does, so contributions agree to 1e-12 like the dense batched predictor's; every other output bit for bit"""
    if pt == 3:
        np.testing.assert_allclose(got, single, rtol=0, atol=1e-12, err_msg=msg)
    else:
        np.testing.assert_array_equal(got, single, err_msg=msg)


def _models(capi):
    rng = np.random.default_rng(41)
    n, F = 4000, 16
    X, z = _model_data(rng, n, F)
    out = {}
    out["binary"] = _train(capi, X, (z > np.median(z)).astype(np.float64), "objective=binary")
    out["multiclass"] = _train(capi, X, np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])).astype(np.float64), "objective=multiclass num_class=3")
    out["regression_nan_missing"] = _train(capi, X, z, "objective=regression")
    out["regression_zero_missing"] = (capi.Booster(model_str=_zero_missing(out["regression_nan_missing"][0].save_model_to_string())), None)
    Xc = X.copy()
    Xc[:, 3] = rng.integers(0, 9, n)
    Xc[rng.random(n) < 0.05, 3] = np.nan
    zc = z + np.array([2, -1, 0, 1.5, -2, 0.5, 1, -0.5, 3])[np.nan_to_num(Xc[:, 3]).astype(int)]
    out["categorical"] = _train(capi, Xc, zc, "objective=regression categorical_feature=3", DS + " categorical_feature=3")
    out["rf"] = _train(capi, X, z, "objective=regression boosting_type=rf bagging_fraction=0.7 bagging_freq=1 feature_fraction=0.8")
    return out, F


def _nasty_csr(rng, n, F):
    """CSR rows over the model's F features and beyond, and their densified [n][F] form (last of repeated indices wins)"""
    indptr, indices, data = [0], [], []
    dense = np.zeros((n, F))
    for r in range(n):
        kind = r % 7
        if kind == 0:
            k = 0                                                            # empty row
        else:
            k = int(rng.integers(1, 2 * F))
        idx = rng.integers(-3, F + 6, k)                                     # negative and past the model's features
        if kind == 2:
            idx = np.sort(idx)
        if kind == 3 and k > 1:
            idx[-1] = idx[0]                                                 # a repeated index
        if kind == 4:
            idx = np.concatenate([idx, idx[::-1]])                           # every index repeated, in reverse order
        val = rng.standard_normal(len(idx))
        val[rng.random(len(idx)) < 0.2] = 0.0                                # stored zeros
        val[rng.random(len(idx)) < 0.1] = np.nan                             # stored NaN
        for j, v in zip(idx, val):
            if 0 <= j < F:
                dense[r, j] = v
        indices.extend(idx.tolist()); data.extend(val.tolist()); indptr.append(len(indices))
    return np.array(indptr, dtype=np.int64), np.array(indices, dtype=np.int32), np.array(data), dense


def _singles(b, indptr, indices, data, num_col, pt, s, k):
    return np.stack([b.predict_for_csr_single(indices[indptr[r]:indptr[r + 1]], data[indptr[r]:indptr[r + 1]], num_col, pt, s, k)
                     for r in range(len(indptr) - 1)])


def test_csr_batch_equals_single_row_and_dense_predictors(built):
    from mmlspark_b200 import capi
    models, F = _models(capi)
    rng = np.random.default_rng(42)
    indptr, indices, data, dense = _nasty_csr(rng, 700, F)
    for name, (b, _) in models.items():
        for num_col in (F, F // 2):
            ip = indptr.astype(np.int32) if num_col == F else indptr        # INT32 and INT64 indptr
            for pt in (capi.PREDICT_NORMAL, capi.PREDICT_RAW_SCORE, capi.PREDICT_LEAF_INDEX, capi.PREDICT_CONTRIB):
                for s, k in RANGES:
                    got = b.predict_csr_device(ip, indices, data, num_col, pt, s, k)
                    _assert_like_single(got, _singles(b, indptr, indices, data, num_col, pt, s, k), pt, "%s %d %d %d" % (name, pt, s, k))
                    np.testing.assert_array_equal(got, b.predict_device(dense, pt, s, k), err_msg="%s %d %d %d" % (name, pt, s, k))


def test_scipy_input_empty_batch_and_stumps(built):
    from mmlspark_b200 import capi
    import scipy.sparse as sp
    rng = np.random.default_rng(43)
    X, z = _model_data(rng, 3000, 8)
    b, _ = _train(capi, X, z, "objective=regression")
    S = sp.csr_matrix(np.nan_to_num(X[:100], nan=0.5))
    np.testing.assert_array_equal(b.predict_csr_device(S), b.predict_device(S.toarray()))
    out = b.predict_csr_device(np.zeros(1, dtype=np.int32), np.zeros(0, dtype=np.int32), np.zeros(0), 8)
    assert out.shape[0] == 0
    # a constant label grows stumps only: no split feature, so no slots (U = 0)
    st, _ = _train(capi, X, np.full(3000, 2.5), "objective=regression", iters=4)
    for pt in (capi.PREDICT_NORMAL, capi.PREDICT_LEAF_INDEX, capi.PREDICT_CONTRIB):
        np.testing.assert_array_equal(st.predict_csr_device(S, predict_type=pt), st.predict_device(S.toarray(), pt))
    # an empty iteration range: no tree is walked
    np.testing.assert_array_equal(b.predict_csr_device(S, predict_type=capi.PREDICT_RAW_SCORE, start_iteration=50),
                                  b.predict_device(S.toarray(), capi.PREDICT_RAW_SCORE, 50))


def test_contrib_over_several_output_chunks(built):
    """50K rows x 2,000 columns x 3 classes: 48 KB of contributions per row, more than one 1 GB output chunk"""
    from mmlspark_b200 import capi
    rng = np.random.default_rng(44)
    n, F, per_row = 50_000, 2000, 20
    cols = rng.integers(0, F // per_row, (n, per_row)) + np.arange(per_row)[None, :] * (F // per_row)      # distinct, ascending
    indptr = (np.arange(n + 1) * per_row).astype(np.int64)
    indices, data = cols.reshape(-1).astype(np.int32), rng.standard_normal(n * per_row)
    dense = np.zeros((n, F))
    dense[np.repeat(np.arange(n), per_row), indices] = data
    y = np.digitize(dense[:, :50].sum(axis=1), [-1.0, 1.0]).astype(np.float32)
    ds = capi.Dataset.from_csr(indptr, indices, data, F, DS)
    ds.set_field("label", y)
    b = capi.Booster(ds, "objective=multiclass num_class=3 num_leaves=15 verbosity=-1 min_data_in_leaf=5")
    for _ in range(6):
        b.update_one_iter()
    got = b.predict_csr_device(indptr, indices, data, F, capi.PREDICT_CONTRIB)
    assert got.shape == (n, 3 * (F + 1)) and 3 * (F + 1) * 8 * n > 2 * (1 << 30)
    np.testing.assert_array_equal(got, b.predict_device(dense, capi.PREDICT_CONTRIB))
    for r in np.concatenate([rng.choice(n, 20, replace=False), [0, n - 1]]):
        _assert_like_single(got[r], b.predict_for_csr_single(indices[indptr[r]:indptr[r + 1]], data[indptr[r]:indptr[r + 1]], F,
                                                             capi.PREDICT_CONTRIB), capi.PREDICT_CONTRIB)


def test_wide_hashed_columns_predict_without_densifying(built):
    """2^18 hashed columns, the shape of test_from_csr_wide_sparse_does_not_densify: train and predict every row on the GPU"""
    from mmlspark_b200 import capi
    rng = np.random.default_rng(29)
    n, F, per_row = 50_000, 1 << 18, 12
    cols = np.sort(rng.integers(0, 4000, (n, per_row)), axis=1) + np.arange(per_row)[None, :] * 4000
    indices = cols.reshape(-1).astype(np.int32)
    indptr = (np.arange(n + 1) * per_row).astype(np.int32)
    data = rng.standard_normal(n * per_row)
    y = (data.reshape(n, per_row)[:, :3].sum(axis=1) + 0.5 * (cols[:, 0] % 2) > 0).astype(np.float32)
    ds = capi.Dataset.from_csr(indptr, indices, data, F, DS)
    ds.set_field("label", y)
    b = capi.Booster(ds, "objective=binary num_leaves=31 verbosity=-1 min_data_in_leaf=5")
    for _ in range(10):
        b.update_one_iter()
    sample = rng.choice(n, 200, replace=False)
    for pt in (capi.PREDICT_NORMAL, capi.PREDICT_RAW_SCORE, capi.PREDICT_LEAF_INDEX):
        got = b.predict_csr_device(indptr, indices, data, F, pt)
        assert got.shape[0] == n
        for r in sample:
            np.testing.assert_array_equal(got[r], b.predict_for_csr_single(indices[indptr[r]:indptr[r + 1]], data[indptr[r]:indptr[r + 1]], F, pt))
    few = np.sort(sample[:16])                                               # contributions stay dense: 2 MB per row at this width
    sub_ptr = np.concatenate([[0], np.cumsum(np.diff(indptr)[few])])
    sub_idx = np.concatenate([indices[indptr[r]:indptr[r + 1]] for r in few])
    sub_val = np.concatenate([data[indptr[r]:indptr[r + 1]] for r in few])
    got = b.predict_csr_device(sub_ptr, sub_idx, sub_val, F, capi.PREDICT_CONTRIB)
    _assert_like_single(got, _singles(b, sub_ptr, sub_idx, sub_val, F, capi.PREDICT_CONTRIB, 0, -1), capi.PREDICT_CONTRIB)
