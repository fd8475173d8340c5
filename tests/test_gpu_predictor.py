"""The device predictor's forest follows the model it predicts: after DART changes the leaf values of trees already on the device, and
after a merge adds trees, the dense and CSR batched predictors equal the host predictor bit for bit.  Dense rows given as a device
pointer predict exactly as the same rows given as a host array, and as the host predictor, for every predict type."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS = "max_bin=255 min_data_in_leaf=5 is_pre_partition=True num_threads=0"
TYPES = ("PREDICT_NORMAL", "PREDICT_RAW_SCORE", "PREDICT_LEAF_INDEX", "PREDICT_CONTRIB")


def _data(seed, n=4000, F=10):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, F))
    X[rng.random((n, F)) < 0.05] = np.nan
    z = np.nan_to_num(X[:, 0]) * 2 - np.nan_to_num(X[:, 1]) + np.nan_to_num(X[:, 2]) ** 2 + 0.3 * rng.standard_normal(n)
    return X, z


def _booster(capi, X, y, params):
    ds = capi.Dataset.from_mat(X, DS)
    ds.set_field("label", y.astype(np.float32))
    return capi.Booster(ds, params + " num_leaves=15 learning_rate=0.2 min_data_in_leaf=5 verbosity=-1"), ds


def _assert_device_equals_host(capi, b, X, pts, msg):
    """predict_device and predict_csr_device on X (densified CSR: every value stored) equal predict_for_mat bit for bit"""
    ptr = (np.arange(X.shape[0] + 1) * X.shape[1]).astype(np.int64)
    idx = np.tile(np.arange(X.shape[1], dtype=np.int32), X.shape[0])
    for pt in pts:
        host = b.predict_for_mat(X, pt)
        np.testing.assert_array_equal(b.predict_device(X, pt), host, err_msg="%s dense %d" % (msg, pt))
        np.testing.assert_array_equal(b.predict_csr_device(ptr, idx, X.ravel(), X.shape[1], pt), host, err_msg="%s csr %d" % (msg, pt))


@pytest.mark.parametrize("objective", ["objective=binary", "objective=multiclass num_class=3"])
def test_dart_changes_to_uploaded_trees_reach_the_device_forest(built, objective):
    """DART negates the dropped trees when the training score is asked for (get_predict(0) here): the tree count stays while earlier
    leaf values change, so a forest kept from the previous call predicts wrong values.  Only this drop path can show a stale forest: the
    re-normalisation always follows a new tree, whose count alone makes the next call upload the forest again."""
    from mmlspark_b200 import capi
    X, z = _data(51)
    y = (z > np.median(z)) if "binary" in objective else np.digitize(z, np.quantile(z, [1 / 3, 2 / 3]))
    b, _ = _booster(capi, X, y, objective + " boosting_type=dart drop_rate=0.5 skip_drop=0.0 max_drop=3")
    rows = X[np.random.default_rng(52).choice(len(X), 300, replace=False)]
    pts = (capi.PREDICT_NORMAL, capi.PREDICT_RAW_SCORE)
    for it in range(8):
        b.update_one_iter()
        _assert_device_equals_host(capi, b, rows, pts, "iteration %d" % it)
        b.get_predict(0)                 # drops trees for the training score: their leaf values change, the tree count does not
        _assert_device_equals_host(capi, b, rows, pts, "iteration %d after the drop" % it)
    shr = {round(float(ln.split("=")[1]), 12) for ln in b.save_model_to_string().split("\n") if ln.startswith("shrinkage=")}
    assert len(shr) > 2                  # trees were dropped and re-normalised


def test_merge_reaches_the_device_forest(built):
    from mmlspark_b200 import capi
    X, z = _data(53)
    a, _ = _booster(capi, X, z, "objective=regression")
    o, _ = _booster(capi, X, -z, "objective=regression")
    for _ in range(5):
        a.update_one_iter()
    for _ in range(3):
        o.update_one_iter()
    rows = X[:500]
    pts = (capi.PREDICT_NORMAL, capi.PREDICT_RAW_SCORE, capi.PREDICT_LEAF_INDEX)
    _assert_device_equals_host(capi, a, rows, pts, "before the merge")
    a.merge(o)
    assert a.predict_device(rows, capi.PREDICT_LEAF_INDEX).shape == (len(rows), 8)
    _assert_device_equals_host(capi, a, rows, pts, "after the merge")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_device_pointer_input_equals_host_input(built, dtype):
    from mmlspark_b200 import capi
    X, z = _data(54)
    b, _ = _booster(capi, X, np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])), "objective=multiclass num_class=3")
    for _ in range(6):
        b.update_one_iter()
    rows = np.ascontiguousarray(X[:700], dtype=dtype)
    nrow, ncol = rows.shape
    buf = capi.DeviceBuffer(rows.nbytes)
    try:
        capi.memcpy(buf.ptr, rows.ctypes.data, rows.nbytes)
        code = capi.DTYPE_FLOAT32 if dtype == np.float32 else capi.DTYPE_FLOAT64
        for name in TYPES:
            pt = getattr(capi, name)
            for s, k in ((0, -1), (2, 3)):
                want = b.predict_device(rows, pt, s, k)
                out = np.full(want.size, np.nan)
                n, ms = C.c_int64(0), C.c_double(0)
                capi.check(capi.load().B200GBM_BoosterPredictForMatDevice(
                    b.handle, buf.ptr, C.c_int(code), C.c_int64(nrow), C.c_int32(ncol), C.c_int(pt), C.c_int(s), C.c_int(k), C.byref(n),
                    out.ctypes.data_as(C.POINTER(C.c_double)), C.byref(ms)))
                assert n.value == want.size
                np.testing.assert_array_equal(out.reshape(want.shape), want, err_msg="%s %d %d" % (name, s, k))
                host = b.predict_for_mat(rows, pt, s, k)      # the host predictor: TreeSHAP there does not fuse multiply-adds
                if pt == capi.PREDICT_CONTRIB:
                    np.testing.assert_allclose(want, host, rtol=0, atol=1e-12, err_msg="%s %d %d" % (name, s, k))
                else:
                    np.testing.assert_array_equal(want, host, err_msg="%s %d %d" % (name, s, k))
    finally:
        buf.free()
