"""Prediction early stopping on the device (k_predict_raw_es behind B200GBM_BoosterPredictFor{Mat,CSR}DeviceWithParameter) against the host
predictor with the same parameter string and the NumPy restatement pred_early_stop_ref, on models the engine trains: binary over 1000
iterations, multiclass with K = 3, 10 and 40 (one lane per class, a group of 16 lanes, a warp walking two classes per lane),
multiclassova, lambdarank, an rf binary model and DART.

Bars: every normal and raw output of the dense predictor (float64 and float32 rows, host and device pointers) and of the CSR predictor
equals the host predictor's bit for bit, and raw scores equal the restatement bit for bit.  Without the key, with pred_early_stop=false
and with a NULL parameter, outputs equal the entry points without a parameter; a margin no row reaches and a period longer than the
range give the same outputs as no key.  Other objectives ignore the keys, the checks fail the call and leave the booster usable, and a
model reloaded from its text predicts the same."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import pred_early_stop_ref as E

pytestmark = pytest.mark.gpu

DS = "max_bin=63 min_data_in_bin=3 bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=7 min_data_in_leaf=10 learning_rate=0.1 verbosity=-1 " + DS
NORMAL_RAW = (0, 1)

# name: (objective params, classes of the labels, iterations)
MODELS = {
    "binary": ("objective=binary", 2, 1000),
    "multiclass3": ("objective=multiclass num_class=3", 3, 60),
    "multiclass10": ("objective=multiclass num_class=10", 10, 30),
    "multiclass40": ("objective=multiclass num_class=40", 40, 12),
    "multiclassova": ("objective=multiclassova num_class=3", 3, 40),
    "lambdarank": ("objective=lambdarank", 4, 60),
    "rf": ("objective=binary boosting=rf bagging_fraction=0.7 bagging_freq=1", 2, 60),
    "dart": ("objective=binary boosting=dart drop_rate=0.2", 2, 60),
}


@pytest.fixture(scope="module")
def capi(built):
    from mmlspark_b200 import capi as c
    c.load()
    return c


def _data(n, seed, classes):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 6))
    X[::11, 2] = np.nan
    z = 2 * X[:, 0] + np.sin(2 * X[:, 1]) + X[:, 3] * X[:, 4] + 0.3 * rng.standard_normal(n)
    y = np.digitize(z, np.quantile(z, np.arange(1, classes) / classes)).astype(np.float32)
    return X, y


def _train(capi, name, extra=""):
    params, classes, iters = MODELS[name]
    X, y = _data(4000, 3, classes)
    ds = capi.Dataset.from_mat(X, DS).set_field("label", y)
    if name == "lambdarank":
        ds.set_field("group", np.full(40, 100, np.int32))
    b = capi.Booster(ds, params + " " + BASE + " " + extra)
    for _ in range(iters):
        b.update_one_iter()
    return b


@pytest.fixture(scope="module")
def models(capi):
    return {name: _train(capi, name).save_model_to_string() for name in MODELS}


def _trees(text):
    from mmlspark_b200.modeltext import parse_model
    return parse_model(text)["trees"]


def _es(freq, margin, on="true"):
    return "pred_early_stop=%s pred_early_stop_freq=%s pred_early_stop_margin=%s" % (on, freq, margin)


def _device_pointer(capi, b, X, pt, s, k, parameter):
    buf = capi.DeviceBuffer(X.nbytes)
    try:
        capi.memcpy(buf.ptr, X.ctypes.data, X.nbytes)
        n = C.c_int64(0)
        capi.check(capi.load().LGBM_BoosterCalcNumPredict(b.handle, C.c_int(X.shape[0]), C.c_int(pt), C.c_int(s), C.c_int(k), C.byref(n)))
        out = np.full(n.value, np.nan)
        code = capi.DTYPE_FLOAT32 if X.dtype == np.float32 else capi.DTYPE_FLOAT64
        capi.check(capi.load().B200GBM_BoosterPredictForMatDeviceWithParameter(
            b.handle, buf.ptr, C.c_int(code), C.c_int64(X.shape[0]), C.c_int32(X.shape[1]), C.c_int(pt), C.c_int(s), C.c_int(k),
            None if parameter is None else parameter.encode(), C.byref(n), out.ctypes.data_as(C.POINTER(C.c_double)), None))
        return out.reshape(X.shape[0], -1)
    finally:
        buf.free()


def _old_device(capi, b, X, pt, s, k):
    """the entry point without a parameter: today's path"""
    n = C.c_int64(0)
    capi.check(capi.load().LGBM_BoosterCalcNumPredict(b.handle, C.c_int(X.shape[0]), C.c_int(pt), C.c_int(s), C.c_int(k), C.byref(n)))
    out = np.full(n.value, np.nan)
    code = capi.DTYPE_FLOAT32 if X.dtype == np.float32 else capi.DTYPE_FLOAT64
    capi.check(capi.load().B200GBM_BoosterPredictForMatDevice(
        b.handle, X.ctypes.data_as(C.c_void_p), C.c_int(code), C.c_int64(X.shape[0]), C.c_int32(X.shape[1]), C.c_int(pt), C.c_int(s),
        C.c_int(k), C.byref(n), out.ctypes.data_as(C.POINTER(C.c_double)), None))
    return out.reshape(X.shape[0], -1)


def _all_device(capi, b, X, pt, s, k, p):
    """host predictor output, after checking every device path against it bit for bit"""
    host = b.predict_for_mat(X, pt, s, k, parameter=p)
    X32 = X.astype(np.float32)
    host32 = b.predict_for_mat(X32.astype(np.float64), pt, s, k, parameter=p)
    for what, got, want in (("f64", b.predict_device(X, pt, s, k, parameter=p), host),
                            ("f32", b.predict_device(X32, pt, s, k, parameter=p), host32),
                            ("f64 device", _device_pointer(capi, b, X, pt, s, k, p), host),
                            ("f32 device", _device_pointer(capi, b, X32, pt, s, k, p), host32),
                            ("csr", b.predict_csr_device(sp.csr_matrix(X), predict_type=pt, start_iteration=s, num_iteration=k, parameter=p), host)):
        np.testing.assert_array_equal(got, want, err_msg="%s type %d range %d,%d %s" % (what, pt, s, k, p))
    return host


CASES = [(10, 2.0, 0, -1), (10, 5.0, 0, -1), (10, 10.0, 0, -1), (3, 1.0, 2, 7), (1, 0.0, 0, -1), (7, 3.0, 1, -1)]


@pytest.mark.parametrize("name", list(MODELS))
def test_device_equals_host_and_restatement(capi, models, name):
    text = models[name]
    b = capi.Booster(model_str=text)
    trees = _trees(text)
    K = b.num_model_per_iteration()
    X, _ = _data(300, 17, 2)
    stopped = 0
    for freq, margin, s, k in CASES:
        p = _es(freq, margin)
        for pt in NORMAL_RAW:
            _all_device(capi, b, X, pt, s, k, p)
        raw = b.predict_device(X, 1, s, k, parameter=p)
        want, walked = E.raw_scores(trees, X[:120], K, s, k, freq, margin, average=name == "rf")
        np.testing.assert_array_equal(raw[:120], want, err_msg="%s %r" % (name, (freq, margin, s, k)))
        t1 = len(trees) // K
        stopped += int((walked < min(t1 - s, k if k > 0 else t1)).sum())
    assert stopped > 0, "no row stopped early: the cases do not exercise the early-stopping kernel"


def test_binary_stops_most_rows_early(capi, models):
    b = capi.Booster(model_str=models["binary"])
    X, _ = _data(200, 5, 2)
    _, walked = E.raw_scores(_trees(models["binary"]), X, 1, freq=10, margin_threshold=5.0)
    assert (walked < 1000).mean() > 0.5
    np.testing.assert_array_equal(b.predict_device(X, 1, parameter=_es(10, 5.0)), b.predict_for_mat(X, 1, parameter=_es(10, 5.0)))


@pytest.mark.parametrize("name", ["binary", "multiclass10"])
def test_chunked_inputs(capi, models, name):
    """4096 float64 columns: 16384 rows per dense chunk; 1000 stored entries per CSR row: two CSR chunks of at most 2^25 entries"""
    b = capi.Booster(model_str=models[name])
    n = 40000
    X = np.zeros((n, 4096))
    X[:, :6], _ = _data(n, 23, 2)
    p = _es(10, 2.0)
    indptr = np.arange(n + 1, dtype=np.int64) * 1000
    indices = np.tile(np.arange(1000, dtype=np.int32), n)
    data = np.ascontiguousarray(X[:, :1000]).ravel()
    for pt in NORMAL_RAW:
        host = b.predict_for_mat(X[:, :6], pt, parameter=p)
        assert (host != b.predict_for_mat(X[:, :6], pt)).any()
        np.testing.assert_array_equal(b.predict_device(X, pt, parameter=p), host)
        np.testing.assert_array_equal(b.predict_csr_device(indptr, indices, data, 4096, pt, parameter=p), host)


@pytest.mark.parametrize("name", ["binary", "multiclass3", "multiclass40", "rf"])
def test_off_and_unreached_settings_equal_todays_path(capi, models, name):
    b = capi.Booster(model_str=models[name])
    X, _ = _data(500, 29, 2)
    iters = b.num_total_model() // b.num_model_per_iteration()
    for pt in NORMAL_RAW:
        for s, k in ((0, -1), (3, 5)):
            today = _old_device(capi, b, X, pt, s, k)
            for p in ("", None, _es(10, 10.0, on="false"), _es(0, -1.0, on="false"), _es(10, 1e300), _es(iters + 1, 0.0)):
                np.testing.assert_array_equal(b.predict_device(X, pt, s, k, parameter=p), today, err_msg=str(p))
                np.testing.assert_array_equal(_device_pointer(capi, b, X, pt, s, k, p), today, err_msg=str(p))
                np.testing.assert_array_equal(b.predict_csr_device(sp.csr_matrix(X), predict_type=pt, start_iteration=s, num_iteration=k,
                                                                   parameter=p), today, err_msg=str(p))
                np.testing.assert_array_equal(b.predict_for_mat(X, pt, s, k, parameter=p), today, err_msg=str(p))


def test_leaf_and_contributions_ignore_the_keys(capi, models):
    b = capi.Booster(model_str=models["multiclass3"])
    X, _ = _data(200, 31, 2)
    for pt in (2, 3):
        want = b.predict_device(X, pt)
        for p in (_es(1, 0.0), _es(0, -1.0)):
            np.testing.assert_array_equal(b.predict_device(X, pt, parameter=p), want)
            np.testing.assert_array_equal(b.predict_csr_device(sp.csr_matrix(X), predict_type=pt, parameter=p), b.predict_csr_device(sp.csr_matrix(X), predict_type=pt))


@pytest.mark.parametrize("objective", ["objective=regression", "objective=cross_entropy"])
def test_other_objectives_ignore_the_keys(capi, objective):
    X, y = _data(3000, 37, 2)
    ds = capi.Dataset.from_mat(X, DS).set_field("label", y)
    b = capi.Booster(ds, objective + " " + BASE)
    for _ in range(20):
        b.update_one_iter()
    Xt, _ = _data(300, 41, 2)
    text = b.save_model_to_string()
    # the same trees under a custom objective (a booster trained on custom gradients) and without an objective line
    name = objective.split("=")[1]
    custom = text.replace("objective=" + name + "\n", "objective=custom\n", 1)
    none = text.replace("objective=" + name + "\n", "", 1)
    assert custom != text and none != text
    for m in (b, capi.Booster(model_str=custom), capi.Booster(model_str=none)):
        for pt in NORMAL_RAW:
            want = m.predict_device(Xt, pt)
            for p in (_es(1, 0.0), _es(0, 1.0), _es(5, "nan")):
                np.testing.assert_array_equal(m.predict_device(Xt, pt, parameter=p), want)
                np.testing.assert_array_equal(m.predict_csr_device(sp.csr_matrix(Xt), predict_type=pt, parameter=p), want)
                np.testing.assert_array_equal(m.predict_for_mat(Xt, pt, parameter=p), want)


@pytest.mark.parametrize("bad,message", [(_es(0, 5.0), "Check failed: (early_stop_freq) > (0)"),
                                         (_es(10, -1.0), "Check failed: (early_stop_margin) >= (0)"),
                                         (_es(10, "nan"), "Check failed: (early_stop_margin) >= (0)")])
def test_checks_fail_and_leave_the_booster_usable(capi, models, bad, message):
    b = capi.Booster(model_str=models["multiclass3"])
    X, _ = _data(100, 47, 2)
    want = b.predict_device(X, 0)
    pattern = message.replace("(", r"\(").replace(")", r"\)")
    with pytest.raises(capi.LightGBMError, match=pattern):
        b.predict_device(X, 0, parameter=bad)
    with pytest.raises(capi.LightGBMError, match=pattern):
        b.predict_csr_device(sp.csr_matrix(X), predict_type=1, parameter=bad)
    np.testing.assert_array_equal(b.predict_device(X, 0), want)
    np.testing.assert_array_equal(b.predict_device(X, 0, parameter=_es(10, 0.5)), b.predict_for_mat(X, 0, parameter=_es(10, 0.5)))


def test_training_booster_keys_do_not_reach_prediction_and_reload_predicts_the_same(capi):
    b = _train(capi, "multiclass3", "pred_early_stop=true pred_early_stop_freq=1 pred_early_stop_margin=0")
    text = b.save_model_to_string()
    assert "pred_early_stop" not in text
    X, _ = _data(300, 53, 2)
    want, _ = E.raw_scores(_trees(text), X[:50], 3, freq=None)
    np.testing.assert_array_equal(b.predict_device(X[:50], 1), want)
    p = _es(5, 1.0)
    r = capi.Booster(model_str=text)
    for pt in NORMAL_RAW:
        np.testing.assert_array_equal(r.predict_device(X, pt, parameter=p), b.predict_device(X, pt, parameter=p))
        np.testing.assert_array_equal(r.predict_for_mat(X, pt, parameter=p), b.predict_device(X, pt, parameter=p))
