"""Sparse features without a GPU: how the estimators resolve `matrixType` and convert the features column, Frame row selection on a
scipy.sparse column, and the argument checks of B200GBM_BoosterPredictForCSRDevice, which run before any device work."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "oracle_golden.json")))


def _dense():
    X = np.array([[0.0, 1.5, np.nan, 0.0],
                  [-0.0, 0.0, 0.0, 0.0],
                  [2.0, 0.0, -3.0, np.nan]])
    return X


def test_to_sparse_keeps_nan_and_drops_zeros():
    from mmlspark_b200.lightgbm.estimators import resolve_matrix_type
    X = _dense()
    m = resolve_matrix_type("sparse", X)
    assert sp.issparse(m) and m.shape == X.shape
    np.testing.assert_array_equal(m.indptr, [0, 2, 2, 5])           # the -0.0 and 0.0 entries are dropped, as != 0 drops them
    np.testing.assert_array_equal(m.indices, [1, 2, 0, 2, 3])
    np.testing.assert_array_equal(m.data, [1.5, np.nan, 2.0, -3.0, np.nan])


def test_matrix_type_resolution():
    from mmlspark_b200.lightgbm.estimators import resolve_matrix_type
    X = _dense()
    S = sp.csr_matrix(np.nan_to_num(X, nan=7.0))
    assert resolve_matrix_type("auto", X) is X                      # dense input keeps its array: the dense path is untouched
    assert resolve_matrix_type("dense", X) is X
    a = resolve_matrix_type("auto", S)
    assert sp.issparse(a) and (a != S).nnz == 0
    d = resolve_matrix_type("dense", S)
    assert isinstance(d, np.ndarray)
    np.testing.assert_array_equal(d, S.toarray())
    assert resolve_matrix_type("sparse", S.tocoo()).format == "csr"
    # repeated entries of a scipy matrix mean their sum, in the sparse and in the densified column alike
    dup = sp.csr_matrix((np.array([1.0, 2.0, 5.0]), np.array([3, 3, 0]), np.array([0, 2, 3])), shape=(2, 4))
    np.testing.assert_array_equal(resolve_matrix_type("auto", dup).toarray(), [[0, 0, 0, 3.0], [5.0, 0, 0, 0]])
    np.testing.assert_array_equal(resolve_matrix_type("dense", dup), [[0, 0, 0, 3.0], [5.0, 0, 0, 0]])
    for bad in ("Sparse", "csr", ""):
        with pytest.raises(ValueError, match="^Invalid parameter matrix type specified: %s$" % bad):
            resolve_matrix_type(bad, X)


def test_invalid_matrix_type_fails_the_fit():
    from mmlspark_b200.lightgbm import Frame, LightGBMRegressor
    df = Frame({"features": sp.csr_matrix(np.eye(6)), "label": np.arange(6.0)})
    with pytest.raises(ValueError, match="Invalid parameter matrix type specified: bogus"):
        LightGBMRegressor(matrixType="bogus", numTasks=1).fit(df)


def test_frame_rows_with_a_sparse_column():
    from mmlspark_b200.lightgbm import Frame
    rng = np.random.default_rng(3)
    X = rng.standard_normal((12, 5)) * (rng.random((12, 5)) < 0.3)
    f = Frame.of({"features": sp.csr_matrix(X), "label": np.arange(12.0), "valid": np.arange(12) % 3 == 0})
    assert sp.issparse(f["features"]) and f.num_rows() == 12
    mask = f["valid"]
    for sel, want in ((slice(2, 7), np.arange(2, 7)), (mask, np.nonzero(mask)[0]), (~mask, np.nonzero(~mask)[0]),
                      (np.array([11, 0, 4, 4]), np.array([11, 0, 4, 4]))):
        part = f.rows(sel)
        assert part.num_rows() == len(want)
        np.testing.assert_array_equal(part["features"].toarray(), X[want])
        np.testing.assert_array_equal(part["label"], want.astype(np.float64))
    coo = Frame({"features": sp.coo_matrix(X), "label": np.arange(12.0)})
    np.testing.assert_array_equal(coo.rows(np.array([5, 1]))["features"].toarray(), X[[5, 1]])
    assert Frame({"features": sp.csr_matrix((0, 5))}).num_rows() == 0


@pytest.fixture(scope="module")
def capi(built):
    from mmlspark_b200 import capi
    capi.load()
    return capi


def _has_gpu():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout.count("GPU ") > 0
    except Exception:
        return False


def _predict_csr(capi, b, indptr, indptr_type, data_type=None, nelem=None):
    indices = np.zeros(8, dtype=np.int32)
    data = np.ones(8, dtype=np.float64)
    out = np.zeros(64, dtype=np.float64)
    n = C.c_int64(0)
    ms = C.c_double(0)
    return capi.load().B200GBM_BoosterPredictForCSRDevice(
        b.handle, capi._ptr(indptr), C.c_int(indptr_type), capi._ptr(indices), capi._ptr(data),
        C.c_int(capi.DTYPE_FLOAT64 if data_type is None else data_type), C.c_int64(len(indptr)), C.c_int64(8 if nelem is None else nelem),
        C.c_int64(4), C.c_int(0), C.c_int(0), C.c_int(-1), C.byref(n), capi._ptr(out), C.byref(ms))


def _error(capi):
    return capi.load().LGBM_GetLastError().decode()


def test_csr_device_predict_checks_arguments_before_device_work(capi):
    """Bad type codes and a bad indptr are rejected on the host, with or without a GPU; the single-row entry clamps instead."""
    b = capi.Booster(model_str=GOLDEN["models"]["binary"]["model"])
    ok32 = np.array([0, 3, 8], dtype=np.int32)
    assert _predict_csr(capi, b, ok32, capi.DTYPE_FLOAT32) == -1 and "INT32 or INT64" in _error(capi)
    assert _predict_csr(capi, b, ok32, capi.DTYPE_INT32, data_type=capi.DTYPE_FLOAT32) == -1 and "FLOAT64" in _error(capi)
    assert _predict_csr(capi, b, ok32, capi.DTYPE_INT32, data_type=capi.DTYPE_INT32) == -1 and "FLOAT64" in _error(capi)
    assert _predict_csr(capi, b, np.array([0, 5, 3], dtype=np.int32), capi.DTYPE_INT32) == -1 and "decreases at position 2" in _error(capi)
    assert _predict_csr(capi, b, np.array([0, 5, 3], dtype=np.int64), capi.DTYPE_INT64) == -1 and "decreases at position 2" in _error(capi)
    assert _predict_csr(capi, b, np.array([-1, 3], dtype=np.int64), capi.DTYPE_INT64) == -1 and "negative" in _error(capi)
    assert _predict_csr(capi, b, ok32, capi.DTYPE_INT32, nelem=7) == -1 and "nelem" in _error(capi)
    assert _predict_csr(capi, b, np.zeros(0, dtype=np.int32), capi.DTYPE_INT32) == -1 and "nindptr" in _error(capi)
    with pytest.raises(capi.LightGBMError, match="decreases"):
        b.predict_csr_device(np.array([0, 2, 1]), np.array([0, 1]), np.array([1.0, 2.0]), 4)
    b.free()


def test_csr_device_predict_fails_loudly_without_gpu(capi):
    if _has_gpu():
        pytest.skip("a GPU is present")
    b = capi.Booster(model_str=GOLDEN["models"]["binary"]["model"])
    with pytest.raises(capi.LightGBMError) as e:
        b.predict_csr_device(sp.csr_matrix(np.eye(3, b.num_feature())))
    assert "no CUDA device" in str(e.value) and "no CPU fallback" in str(e.value)
    b.free()
